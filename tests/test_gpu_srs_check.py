"""GPU tests of the checked params-file read (ParamsKZG::read_custom, spb_srs_read_file_custom): SPB_SERDE_RAW_BYTES rejects
a non-canonical coordinate or a point off its curve with SPB_ERR_DATA and names the first such point in file order;
SPB_SERDE_RAW_BYTES_UNCHECKED and spb_srs_read_file accept the same files as before.

Valid files: the oracle's gen_srs-style file at k = 9, and a k = 20 file written by the library (ParamsKZG.setup + write), whose
bases span several 16 MiB (2^18-point) staging chunks of the read."""
import contextlib
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.gpu_common import be, device_lists  # noqa: F401

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
X_REASON = "x is not less than the field modulus"
Y_REASON = "y is not less than the field modulus"
CURVE_REASON = "not on the curve"


class SrsFile:
    def __init__(self, path, k):
        self.path, self.k, self.n = path, k, 1 << k

    def g1_offset(self, basis, i):
        return 4 + 64 * (i + (self.n if basis == "g_lagrange" else 0))

    def g2_offset(self, which):
        return 4 + 128 * self.n + (128 if which == "s_g2" else 0)


@pytest.fixture(scope="module")
def k9(orc, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("srs9") / "kzg_bn254_9.srs")
    orc.write_params_file(path, 9)
    return SrsFile(path, 9)


@pytest.fixture(scope="module")
def k20(be, orc, tmp_path_factory):
    from spectre_b200.halo2 import ParamsKZG
    path = str(tmp_path_factory.mktemp("srs20") / "kzg_bn254_20.srs")
    g2 = np.empty((4, 4), dtype=np.uint64); s_g2 = np.empty((4, 4), dtype=np.uint64)
    orc.lib().orc_srs_g2_raw(g2.ctypes.data_as(ctypes.c_void_p), s_g2.ctypes.data_as(ctypes.c_void_p))
    params = ParamsKZG.setup(be, 20, orc.srs_tau())
    params.set_g2(g2, s_g2)
    params.write(path)
    del params
    return SrsFile(path, 20)


def _int(b):
    return int.from_bytes(b, "little")


def _bytes(v):
    return v.to_bytes(32, "little")


# corruptions of one stored 64-byte G1 point (x limbs, then y limbs) -> (new bytes, reason the check must give)
def flip_y_low_bit(pt):
    return pt[:32] + bytes([pt[32] ^ 1]) + pt[33:], CURVE_REASON


def x_plus_p(pt):
    return _bytes(_int(pt[:32]) + P) + pt[32:], X_REASON          # still on the curve mod p


def y_equal_p(pt):
    return pt[:32] + _bytes(P), Y_REASON


CORRUPTIONS = [flip_y_low_bit, x_plus_p, y_equal_p]


@contextlib.contextmanager
def patched(path, edits):
    """edits: [(offset, bytes)] written in place, the original bytes restored afterwards"""
    saved = []
    with open(path, "r+b") as f:
        for off, data in edits:
            f.seek(off); saved.append((off, f.read(len(data))))
            f.seek(off); f.write(data)
    try:
        yield
    finally:
        with open(path, "r+b") as f:
            for off, data in saved:
                f.seek(off); f.write(data)


def read_point(path, off, size=64):
    with open(path, "rb") as f:
        f.seek(off)
        return f.read(size)


def checked_read_error(be, path):
    from spectre_b200.halo2 import BackendError, ParamsKZG
    with pytest.raises(BackendError) as ei:
        ParamsKZG.read_custom(be, path, "RawBytes")
    msg = str(ei.value)
    assert "failed (-6)" in msg, msg                                 # SPB_ERR_DATA
    return msg


def assert_unchecked_reads_accept(be, path):
    from spectre_b200.halo2 import ParamsKZG
    for params in (ParamsKZG.read_custom(be, path, "RawBytesUnchecked"), ParamsKZG.read(be, path)):
        assert params.k == int.from_bytes(read_point(path, 0, 4), "little")


@pytest.mark.parametrize("which", ["k9", "k20"])
def test_checked_read_of_valid_file_matches_unchecked(be, orc, request, which):
    from spectre_b200.halo2 import BASIS_G, BASIS_G_LAGRANGE, ParamsKZG
    f = request.getfixturevalue(which)
    checked = ParamsKZG.read_custom(be, f.path, "RawBytes")
    assert be.last_device_ms > 0.0                                   # the check kernels' device time
    plain = ParamsKZG.read_custom(be, f.path, "RawBytesUnchecked")
    assert checked.k == plain.k == f.k
    for basis in (BASIS_G, BASIS_G_LAGRANGE):
        assert np.array_equal(checked.get_g(basis=basis), plain.get_g(basis=basis))
    assert all(np.array_equal(a, b) for a, b in zip(checked.get_g2(), plain.get_g2()))
    if f.k == 9:
        assert np.array_equal(checked.get_g(basis=BASIS_G), orc.srs_g(9, 0, 512))
    poly = orc.fr_random_chacha(f.n, 0x5c4ec)
    assert np.array_equal(orc.g1_to_affine(checked.commit_lagrange(poly)), orc.commit_lagrange_known_tau(f.k, poly))


POSITIONS = [("k9", "g", 0), ("k9", "g_lagrange", 0), ("k9", "g_lagrange", 511),
             ("k20", "g", (1 << 18) - 1), ("k20", "g", 1 << 18), ("k20", "g", (1 << 20) - 1),
             ("k20", "g_lagrange", 0), ("k20", "g_lagrange", (1 << 20) - 1)]


@pytest.mark.parametrize("which,basis,index", POSITIONS)
def test_one_bad_point_is_named(be, request, which, basis, index):
    """every corruption at every position: the checked read refuses with the basis, index and reason; the unchecked format and
    the plain read accept the file as before"""
    f = request.getfixturevalue(which)
    off = f.g1_offset(basis, index)
    pt = read_point(f.path, off)
    for corrupt in CORRUPTIONS:
        data, reason = corrupt(pt)
        with patched(f.path, [(off, data)]):
            msg = checked_read_error(be, f.path)
            assert ": %s[%d]: %s" % (basis, index, reason) in msg, (corrupt.__name__, msg)
            assert_unchecked_reads_accept(be, f.path)


@pytest.mark.parametrize("which", ["k9", "k20"])
def test_bad_g2_trailer_is_named(be, request, which):
    f = request.getfixturevalue(which)
    s_off = f.g2_offset("s_g2")
    s_g2 = read_point(f.path, s_off, 128)
    bad_s = s_g2[:96] + bytes([s_g2[96] ^ 1]) + s_g2[97:]            # s_g2.y.c1, low bit
    with patched(f.path, [(s_off, bad_s)]):
        assert ": s_g2: " + CURVE_REASON in checked_read_error(be, f.path)
        assert_unchecked_reads_accept(be, f.path)
    g_off = f.g2_offset("g2")
    g2 = read_point(f.path, g_off, 128)
    bad_g = _bytes(_int(g2[:32]) + P) + g2[32:]                       # g2.x.c0 + p
    with patched(f.path, [(g_off, bad_g)]):
        assert ": g2: " + X_REASON in checked_read_error(be, f.path)
        assert_unchecked_reads_accept(be, f.path)
    with patched(f.path, [(g_off, bad_g), (s_off, bad_s)]):           # g2 comes first in the file
        assert ": g2: " + X_REASON in checked_read_error(be, f.path)


def test_identity_is_accepted(be, k9):
    from spectre_b200.halo2 import BASIS_G, ParamsKZG
    with patched(k9.path, [(k9.g1_offset("g", 37), bytes(64))]):
        params = ParamsKZG.read_custom(be, k9.path, "RawBytes")
        assert not params.get_g(37, 1, basis=BASIS_G).any()


def test_first_bad_point_in_file_order(be, k9):
    """bad points at g_lagrange[5] and g[100]: g comes before g_lagrange in the file, so g[100] is reported"""
    edits = []
    for basis, i in (("g_lagrange", 5), ("g", 100)):
        off = k9.g1_offset(basis, i)
        edits.append((off, flip_y_low_bit(read_point(k9.path, off))[0]))
    with patched(k9.path, edits):
        msg = checked_read_error(be, k9.path)
        assert ": g[100]: " + CURVE_REASON in msg and "g_lagrange[5]" not in msg, msg
    with patched(k9.path, edits[:1]):
        assert ": g_lagrange[5]: " + CURVE_REASON in checked_read_error(be, k9.path)


def test_unknown_format_is_an_argument_error(be, k9):
    from spectre_b200.halo2 import ParamsKZG
    for fmt in (0, 3, -1, 1 << 20):
        h = ctypes.c_void_p(0)
        rc = be.lib.spb_srs_read_file_custom(be.ctx, k9.path.encode(), ctypes.c_int(fmt), ctypes.byref(h))
        assert rc == -2 and not h.value, fmt                          # SPB_ERR_ARG, *out untouched
    with pytest.raises(ValueError):
        ParamsKZG.read_custom(be, k9.path, "Processed")


def test_context_reads_a_valid_file_after_a_rejection(be, orc, k9):
    from spectre_b200.halo2 import ParamsKZG
    off = k9.g1_offset("g", 0)
    with patched(k9.path, [(off, x_plus_p(read_point(k9.path, off))[0])]):
        h = ctypes.c_void_p(0)
        rc = be.lib.spb_srs_read_file_custom(be.ctx, k9.path.encode(), ctypes.c_int(1), ctypes.byref(h))
        assert rc == -6 and not h.value                               # *out untouched
    params = ParamsKZG.read_custom(be, k9.path, "RawBytes")
    poly = orc.fr_random_chacha(k9.n, 0xa11)
    assert np.array_equal(orc.g1_to_affine(params.commit_lagrange(poly)), orc.commit_lagrange_known_tau(9, poly))
    assert np.array_equal(orc.g1_to_affine(params.commit(poly)), orc.commit_known_tau(poly))


@pytest.mark.parametrize("ids", device_lists())
def test_several_devices_report_the_global_index(orc, k9, ids):
    """each shard is checked on its own device; a bad point in a shard after the first (on two devices, points 256..511 of
    512) is named by its index in the file"""
    from spectre_b200 import halo2
    be2 = halo2.Backend(ids)
    try:
        for basis, i in (("g", 300), ("g_lagrange", 511), ("g", 255)):
            off = k9.g1_offset(basis, i)
            with patched(k9.path, [(off, flip_y_low_bit(read_point(k9.path, off))[0])]):
                assert ": %s[%d]: %s" % (basis, i, CURVE_REASON) in checked_read_error(be2, k9.path)
        params = halo2.ParamsKZG.read_custom(be2, k9.path, "RawBytes")
        poly = orc.fr_random_chacha(k9.n, 0xd2)
        assert np.array_equal(orc.g1_to_affine(params.commit_lagrange(poly)), orc.commit_lagrange_known_tau(9, poly))
        del params
    finally:
        be2.close()


@pytest.mark.parametrize("which,basis,index", [("k9", "g_lagrange", 511), ("k20", "g", 1 << 18)])
def test_cpp_read_custom(be, request, tmp_path, which, basis, index):
    """include/spectre_b200.hpp's ParamsKZG::read_custom accepts the valid file and refuses a copy with one bad point"""
    from spectre_b200 import build
    f = request.getfixturevalue(which)
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "srs_read_custom")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "srs_read_custom.cpp"),
                           "-L" + libdir, "-lspectre_b200", "-Wl,-rpath," + libdir])
    bad = str(tmp_path / "bad.srs")
    shutil.copyfile(f.path, bad)
    off = f.g1_offset(basis, index)
    with patched(bad, [(off, y_equal_p(read_point(bad, off))[0])]):
        out = subprocess.run([exe, f.path, bad, "%s[%d]: %s" % (basis, index, Y_REASON)], capture_output=True, text=True)
    assert out.returncode == 0 and "read_custom ok k=%d" % f.k in out.stdout, out.stdout + out.stderr
