"""Per-part proving keys (cosets="per_part") on the CPU oracle engine: create_proof evaluates the quotient one n-row coset part
at a time and proves the resident key's bytes; the key and its file are a lean key's; the compiled driver does the same over
the test-only ABI shim; and the part transform's first-pass load and the part scatter run on the CPU (tests/hostemu/per_part.cpp)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from spectre_b200 import circuits, plonk
from spectre_b200.transcript import EvmTranscriptWrite
from tests import plonk_verifier, pyref
from tests.per_part_oracle_engine import PerPartOracleEngine as OracleEngine, permutation_constraints_coset
from tests.plonk_oracle_engine import SeededRng
from tests.test_hostemu import _p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTANCES = [3, 1, 4]


def _case(shape, k):
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, INSTANCES, lookup_bits=3, groups=30)
        return cs, fixed, [adv], copies
    if shape == "wide":
        cs = circuits.wide_shape(3)
        fixed, adv, copies = circuits.wide_witness(cs, k, INSTANCES, lookup_bits=3, groups=20)
        return cs, fixed, adv, copies
    cs = circuits.halo2lib_shape(3, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, INSTANCES, lookup_bits=4, groups=20, num_gate_advice=3, num_lookup_advice=2)
    return cs, fixed, adv, copies


def _prove(E, pk, adv, seed=11):
    return plonk.create_proof(E, pk, [INSTANCES], adv, SeededRng(seed), EvmTranscriptWrite(pk.vk_digest))


def _verify(orc, cs, k, pk, proof):
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    return plonk_verifier.verify(cs, k, pk.vk_digest, pk.fixed_commitments, pk.sigma_commitments, [INSTANCES], proof, tau)


@pytest.mark.parametrize("shape,k", [("aggregation", 6), ("aggregation", 8), ("wide", 7), ("halo2lib", 8)])
def test_per_part_key_proves_the_resident_bytes_and_verifies(orc, shape, k):
    cs, fixed, adv, copies = _case(shape, k)
    E = OracleEngine(k, cs.degree())
    resident = plonk.keygen(E, cs, k, fixed, copies)
    per_part = plonk.keygen(E, cs, k, fixed, copies, cosets="per_part")
    assert per_part.lean and per_part.per_part and not resident.per_part and len(per_part.l_polys) == 3
    assert per_part.fixed_cosets is None and per_part.sigma_cosets is None and per_part.l0 is None
    proof = _prove(E, per_part, adv)
    assert proof == _prove(E, resident, adv)
    assert _prove(E, per_part, adv) == proof                      # the key is unchanged by a proof
    assert _verify(orc, cs, k, per_part, proof)


def _high_degree_shape():
    """a synthetic circuit whose gate has degree 9: R = 8 coset parts (extended_k = k + 3)"""
    A, F, I = plonk.Advice, plonk.Fixed, plonk.Instance
    gate = plonk.Prod(F(0), plonk.Sum(plonk.Prod(plonk.Prod(plonk.Prod(A(0), A(0)), plonk.Prod(A(0), A(0))), plonk.Prod(plonk.Prod(A(0), A(0)), A(0, 1))),
                                      plonk.Neg(plonk.Prod(plonk.Prod(plonk.Prod(A(1), A(1)), plonk.Prod(A(1), A(1))), plonk.Prod(plonk.Prod(A(1), A(1)), A(1, 1))))))
    return plonk.ConstraintSystem(num_fixed=1, num_advice=2, num_instance=1, gates=[gate], lookups=[],
                                  permutation=[("advice", 0), ("advice", 1), ("instance", 0)])


def test_per_part_key_with_eight_parts(orc):
    """degree 9: R = 8. Advice columns 0 and 1 are equal (the gate is zero), the instance is copied into both."""
    k = 6
    cs = _high_degree_shape()
    n = 1 << k
    E = OracleEngine(k, cs.degree())
    assert E.extended_k - k == 3
    usable = n - (cs.blinding_factors() + 1)
    vals = [(i * 7 + 3) % 97 for i in range(usable)]
    vals[:len(INSTANCES)] = INSTANCES
    col = np.zeros((n, 4), dtype=np.uint64)
    col[:usable] = plonk.fr_mont_rows(vals)
    sel = np.zeros((n, 4), dtype=np.uint64)
    sel[:usable - 1] = plonk.fr_mont(1)
    copies = [((2, i), (0, i)) for i in range(len(INSTANCES))] + [((0, i), (1, i)) for i in range(len(INSTANCES))]
    resident = plonk.keygen(E, cs, k, [sel], copies)
    per_part = plonk.keygen(E, cs, k, [sel], copies, cosets="per_part")
    proofs = [plonk.create_proof(E, pk, [INSTANCES], [col, col.copy()], SeededRng(5), EvmTranscriptWrite(pk.vk_digest)) for pk in (resident, per_part)]
    assert proofs[0] == proofs[1]
    assert _verify(orc, cs, k, per_part, proofs[1])


def test_per_part_key_file_is_the_resident_file_and_reads_back_per_part(orc, tmp_path):
    k = 7
    cs, fixed, adv, copies = _case("halo2lib", k)
    E = OracleEngine(k, cs.degree())
    resident = plonk.keygen(E, cs, k, fixed, copies)
    per_part = plonk.keygen(E, cs, k, fixed, copies, cosets="per_part")
    paths = [str(tmp_path / name) for name in ("resident.pkey", "per_part.pkey")]
    plonk.write_pk(E, resident, paths[0])
    plonk.write_pk(E, per_part, paths[1])
    with open(paths[0], "rb") as f1, open(paths[1], "rb") as f2:
        assert f1.read() == f2.read()
    want = _prove(E, resident, adv)
    reads = []
    inner = E.read_from_file
    E.read_from_file = lambda p, offset, rows: reads.append(rows) or inner(p, offset, rows)
    back = plonk.read_pk(E, cs, paths[1], cosets="per_part")
    E.read_from_file = inner
    assert reads == [1 << k] * (2 * (cs.num_fixed + len(cs.permutation)))     # the coset sections are skipped
    assert back.lean and back.per_part and back.fixed_cosets is None and back.l0 is None
    assert _prove(E, back, adv) == want


def test_per_part_key_device_bytes_is_the_lean_formula():
    for cs, k, ek in ((circuits.aggregation_shape(), 24, 26), (circuits.halo2lib_shape(), 20, 22)):
        assert plonk.key_device_bytes(cs, k, ek, "per_part") == plonk.key_device_bytes(cs, k, ek, "on_demand")


def test_part_transforms_are_the_whole_coset_sliced(orc):
    """the engine contract the driver relies on, restated: part j of coeff_to_extended is its rows j, j + R, ...; scattering
    every part back rebuilds the whole coset"""
    k = 5
    E = OracleEngine(k, 5)
    R = 1 << (E.extended_k - k)
    polys = [E.upload(orc.fr_random_chacha(1 << k, 0x5eed0900 + i)) for i in range(3)]
    whole = [E.coeff_to_extended(p).a for p in polys]
    back = E.alloc(1 << E.extended_k)
    outs = [E.alloc(1 << k) for _ in polys]
    for j in range(R):
        E.coeff_to_extended_part_many(polys, j, outs)
        for o, w in zip(outs, whole):
            assert np.array_equal(o.a, w[j::R])
        E.extended_part_scatter(outs[0], j, back)
    assert np.array_equal(back.a, whole[0])


def test_oracle_coset_permutation_row_over_parts(orc):
    """the oracle's coset permutation terms on part j (size n, rot_scale 1, g_j) are the whole-coset terms sliced [j::R]"""
    k, j_deg = 5, 5
    d = orc.Domain(j_deg, k)
    ek, n = d.extended_k, 1 << k
    R, E = 1 << (ek - k), 1 << ek
    rnd = lambda rows, s: orc.fr_random_chacha(rows, 0x5eed0a00 + s)
    z, cols, sig = [rnd(E, 1), rnd(E, 2)], [rnd(E, 3), rnd(E, 4), rnd(E, 5)], [rnd(E, 6), rnd(E, 7), rnd(E, 8)]
    l0, ll, la, vals = rnd(E, 9), rnd(E, 10), rnd(E, 11), rnd(E, 12)
    beta, gamma, y = rnd(1, 13)[0], rnd(1, 14)[0], rnd(1, 15)[0]
    whole = orc.permutation_constraints(vals, R, -3, 2, z, cols, sig, l0, ll, la, beta, gamma, y, d.extended_omega)
    w_ext = pyref.omega(ek)
    for j in range(R):
        g = orc.fr([pyref.ZETA * pow(w_ext, j, pyref.R_MOD) % pyref.R_MOD])[0]
        s = lambda a: np.ascontiguousarray(a[j::R])
        got = permutation_constraints_coset(s(vals), 1, -3, 2, [s(a) for a in z], [s(a) for a in cols], [s(a) for a in sig], s(l0), s(ll), s(la),
                                            beta, gamma, y, g, d.omega)
        assert np.array_equal(got, whole[j::R])
    assert n == whole.shape[0] // R


# ---- hostemu: the kernels' per-element bodies on the CPU ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def he(tmp_path_factory):
    """tests/hostemu/per_part.cpp (hostemu.cpp plus the per-part bodies), 64-bit host arithmetic, built outside the checkout"""
    so = str(tmp_path_factory.mktemp("hostemu") / "libhostemu_per_part.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "hostemu", "per_part.cpp")])
    return ctypes.CDLL(so)


@pytest.mark.parametrize("k,j,max_digit,tile_log,threads,full", [(3, 4, 11, 11, 256, 0), (6, 3, 11, 10, 64, 0), (8, 5, 4, 6, 32, 0), (9, 9, 4, 6, 32, 1),
                                                                 (10, 4, 5, 7, 64, 0), (12, 3, 6, 8, 128, 1)])
def test_hostemu_part_transform_is_the_oracle_coset_sliced(he, orc, k, j, max_digit, tile_log, threads, full):
    """the NTT kernel's phases with the g^a power-table pre-scale, on one-pass and multi-pass plans and with two-level or full
    twiddle tables: every part j equals the oracle's coset sliced [j::R]"""
    d = orc.Domain(j, k)
    ek = d.extended_k
    R = 1 << (ek - k)
    coeff = orc.fr_random_chacha(1 << k, 0x5eed0b00 + k)
    whole = d.coeff_to_extended(coeff)
    w_ext = pyref.omega(ek)
    for part in range(R):
        g = orc.fr([pyref.ZETA * pow(w_ext, part, pyref.R_MOD) % pyref.R_MOD])[0]
        out = np.zeros((1 << k, 4), dtype=np.uint64)
        passes = he.he_ntt_part(_p(coeff), _p(out), ctypes.c_uint32(k), _p(d.omega), _p(np.ascontiguousarray(g)), ctypes.c_uint32(max_digit),
                                ctypes.c_uint32(tile_log), ctypes.c_uint32(threads), ctypes.c_int(full))
        assert passes == max(1, -(-k // max_digit))
        assert np.array_equal(out, whole[part::R]), "part %d of %d" % (part, R)


def test_hostemu_part_scatter(he, orc):
    k, R = 6, 4
    parts = [orc.fr_random_chacha(1 << k, 0x5eed0c00 + j) for j in range(R)]
    ext = np.zeros((R << k, 4), dtype=np.uint64)
    for j, p in enumerate(parts):
        he.he_extended_part_scatter(_p(p), _p(ext), ctypes.c_uint32(j), ctypes.c_uint32(R), ctypes.c_uint64(1 << k))
    for j, p in enumerate(parts):
        assert np.array_equal(ext[j::R], p)


def test_hostemu_coset_permutation_row(he, orc):
    """the kernel's row with (zeta, extended_omega) is the existing row; with (g_j, omega) on a part it is the oracle's"""
    k, jd = 5, 4
    d = orc.Domain(jd, k)
    ek = d.extended_k
    R, E = 1 << (ek - k), 1 << ek
    rnd = lambda rows, s: orc.fr_random_chacha(rows, 0x5eed0d00 + s)
    z, cols, sig = [rnd(E, 1), rnd(E, 2)], [rnd(E, 3), rnd(E, 4), rnd(E, 5)], [rnd(E, 6), rnd(E, 7), rnd(E, 8)]
    l0, ll, la, vals = rnd(E, 9), rnd(E, 10), rnd(E, 11), rnd(E, 12)
    beta, gamma, y = rnd(1, 13)[0], rnd(1, 14)[0], rnd(1, 15)[0]

    def run(fn, values, rot_scale, zz, cc, ss, a0, a1, a2, *tail):
        values = np.ascontiguousarray(values).copy()
        keep = [np.ascontiguousarray(a) for a in zz + cc + ss + [a0, a1, a2]]
        arr = lambda xs: (ctypes.c_void_p * len(xs))(*[x.ctypes.data for x in xs])
        zp, cp, sp = arr(keep[:len(zz)]), arr(keep[len(zz):len(zz) + len(cc)]), arr(keep[len(zz) + len(cc):len(zz) + len(cc) + len(ss)])
        fn(_p(values), ctypes.c_uint64(values.shape[0]), ctypes.c_int32(rot_scale), ctypes.c_int32(-3), ctypes.c_uint32(len(zz)), ctypes.c_uint32(2), zp,
           ctypes.c_uint32(len(cc)), cp, sp, _p(keep[-3]), _p(keep[-2]), _p(keep[-1]), _p(beta), _p(gamma), _p(y), *[_p(np.ascontiguousarray(t)) for t in tail])
        return values
    existing = run(he.he_permutation_constraints, vals, R, z, cols, sig, l0, ll, la, d.extended_omega)
    zeta = orc.fr([pyref.ZETA])[0]
    assert np.array_equal(run(he.he_permutation_constraints_coset, vals, R, z, cols, sig, l0, ll, la, zeta, d.extended_omega), existing)
    w_ext = pyref.omega(ek)
    for j in range(R):
        g = orc.fr([pyref.ZETA * pow(w_ext, j, pyref.R_MOD) % pyref.R_MOD])[0]
        s = lambda a: np.ascontiguousarray(a[j::R])
        got = run(he.he_permutation_constraints_coset, s(vals), 1, [s(a) for a in z], [s(a) for a in cols], [s(a) for a in sig], s(l0), s(ll), s(la), g, d.omega)
        assert np.array_equal(got, existing[j::R])


# ---- the compiled driver in per-part mode over the CPU shim of the C ABI ------------------------------------------------------
def build_per_part_main_over_the_shim(out_dir):
    """tests/cpp/prover_main_per_part.cpp linked against tests/abi_shim/per_part_shim.cpp (the oracle behind the C ABI, with the
    per-part entry points), built into out_dir"""
    from oracle import oracle as orc
    orc.build()
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    shim = os.path.join(out_dir, "libspb_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", shim, os.path.join(ROOT, "tests", "abi_shim", "per_part_shim.cpp"),
                           "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    exe = os.path.join(out_dir, "prover_main_per_part")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "prover_main_per_part.cpp"), "-L" + out_dir, "-lspb_shim",
                           "-Wl,-rpath," + out_dir, "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    return exe


@pytest.mark.parametrize("shape,k", [("aggregation", 7), ("halo2lib", 8)])
def test_cpp_driver_with_a_per_part_key_reproduces_the_python_proof(orc, tmp_path, shape, k):
    from tools import cpp_driver
    exe = build_per_part_main_over_the_shim(str(tmp_path))
    cs, fixed, adv, copies = _case(shape, k)
    digest = 0x1234567890abcdef1234
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest, cosets="per_part")
    rec = cpp_driver.RecordingRng(SeededRng(77))
    proof = plonk.create_proof(E, pk, [INSTANCES], adv, rec, EvmTranscriptWrite(pk.vk_digest))
    case = tmp_path / "case"
    case.mkdir()
    head = "shape aggregation" if shape == "aggregation" else "shape halo2lib 3 2"
    cpp_driver.dump_case(str(case), head, k, digest, INSTANCES, copies, rec.counts, fixed, adv, rec.rows, orc.srs_tau())
    rc, log, cproof, _, _ = cpp_driver.run(exe, str(case), repeat=2)
    assert rc == 0, log
    assert cproof == proof


def test_cpp_driver_without_the_per_part_entry_points_refuses_only_per_part(orc, tmp_path):
    """include/spectre_b200_prover.hpp references the per-part entry points weakly: linked against a build of the C ABI without
    them (tests/abi_shim/shim.cpp alone) the per-part program still links, and its proof fails with an error naming them"""
    from tools import cpp_driver
    orc.build()
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    out = str(tmp_path)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", os.path.join(out, "libspb_shim.so"), os.path.join(ROOT, "tests", "abi_shim", "shim.cpp"),
                           "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    exe = os.path.join(out, "prover_main_per_part")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "prover_main_per_part.cpp"), "-L" + out, "-lspb_shim",
                           "-Wl,-rpath," + out, "-L" + ref_dir, "-lhalo2_oracle", "-Wl,-rpath," + ref_dir])
    k = 7
    cs, fixed, adv, copies = _case("aggregation", k)
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=0x1234, cosets="per_part")
    rec = cpp_driver.RecordingRng(SeededRng(77))
    plonk.create_proof(E, pk, [INSTANCES], adv, rec, EvmTranscriptWrite(pk.vk_digest))
    case = tmp_path / "case"
    case.mkdir()
    cpp_driver.dump_case(str(case), "shape aggregation", k, 0x1234, INSTANCES, copies, rec.counts, fixed, adv, rec.rows, orc.srs_tau())
    rc, log, cproof, _, _ = cpp_driver.run(exe, str(case))
    assert rc != 0 and cproof is None
    assert "spb_coeff_to_extended_part_batch_dev" in log, log
