"""CPU-only tests of the DEVICE arithmetic (spectre_b200/csrc/{ptx,field,curve}.cuh).

The headers are compiled for the host twice by tests/hostemu: with -DSPB_EMULATE_PTX every PTX carry-chain
primitive is emulated (so the exact 32-bit-limb algorithm the GPU runs is what is tested), and without it
the 64-bit host-glue path is tested. Both are compared with Python big integers and with the oracle.
"""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import pyref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu")


def _build(name, flags):
    so = os.path.join(HERE, name)
    src = os.path.join(HERE, "hostemu.cpp")
    hdrs = [os.path.join(HERE, "..", "..", "spectre_b200", "csrc", h) for h in ("ptx.cuh", "field.cuh", "curve.cuh", "msm.cuh", "ntt.cuh", "quotient.cuh")]
    newest = max(os.path.getmtime(p) for p in [src] + hdrs)
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, src])
    return ctypes.CDLL(so)


@pytest.fixture(scope="module", params=["ptx", "native"])
def he(request):
    if request.param == "ptx":
        return _build("libhostemu_ptx.so", ["-DSPB_EMULATE_PTX"])
    return _build("libhostemu_native.so", [])


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _edge_and_random(mod, n, rng):
    vals = [0, 1, 2, mod - 1, mod - 2, (mod - 1) // 2, 1 << 253, (1 << 253) + 12345, 0xFFFFFFFF, 1 << 32, (1 << 64) - 1, 1 << 64,
            (1 << 128) - 1, 1 << 224]
    vals = [v % mod for v in vals]
    vals += [rng.randrange(mod) for _ in range(n - len(vals))]
    return vals


@pytest.mark.parametrize("field", ["fr", "fq"])
def test_mul_and_sqr_carry_patterns(he, orc, field):
    """The interleaved CIOS multiplier (field.cuh fp_mul) and the squarer (fp_sqr: sqr8 then fp_mont_reduce) on operands
    built to stress their carries: halves near 2^128, all-ones limbs, equal halves, single-limb values, and 20000 random
    pairs. The per-site carry coverage of these primitives is checked by tests/test_hostemu_carry_coverage.py."""
    mod = pyref.R_MOD if field == "fr" else pyref.P_MOD
    rng = random.Random(99)
    F = (1 << 128) - 1
    special = [0, 1, mod - 1, mod - 2, F, F << 96, (F << 126) % mod, ((1 << 126) - 1) << 128 | F, (mod >> 128) << 128, mod & F, 0xFFFFFFFF << 96,
               (0xFFFFFFFF << 224) % mod, ((1 << 253) - 1) % mod, (1 << 253) % mod, F | (F >> 3) << 128, 0xFFFFFFFF00000000FFFFFFFF00000000FFFFFFFF00000000FFFFFFFF % mod]
    special += [(((1 << 32) - 1) << (32 * i)) % mod for i in range(8)] + [(1 << (32 * i)) % mod for i in range(8)]
    a = [x for x in special for _ in special] + [rng.randrange(mod) for _ in range(20000)]
    b = [y for _ in special for y in special] + [rng.randrange(mod) for _ in range(20000)]
    rinv = pow(1 << 256, -1, mod)
    A = orc.to_mont(a, mod); B = orc.to_mont(b, mod)
    out = np.empty_like(A)
    n = ctypes.c_size_t(len(a))
    getattr(he, f"he_{field}_mul")(_p(out), _p(A), _p(B), n)
    assert orc.from_mont(out, mod) == [x * y % mod for x, y in zip(a, b)]
    getattr(he, f"he_{field}_sqr")(_p(out), _p(A), n)
    assert orc.from_mont(out, mod) == [x * x % mod for x in a]
    # raw (non-Montgomery) operands exercise other limb patterns: result = a * b * 2^-256
    raw_a = np.array([[(v >> (64 * j)) & (2**64 - 1) for j in range(4)] for v in a], dtype=np.uint64)
    raw_b = np.array([[(v >> (64 * j)) & (2**64 - 1) for j in range(4)] for v in b], dtype=np.uint64)
    getattr(he, f"he_{field}_mul")(_p(out), _p(raw_a), _p(raw_b), n)
    got = [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in out]
    assert got == [x * y * rinv % mod for x, y in zip(a, b)]
    getattr(he, f"he_{field}_sqr")(_p(out), _p(raw_a), n)
    got = [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in out]
    assert got == [x * x * rinv % mod for x in a]


def test_mul_sub_mul_single_reduction(he, orc):
    """a*b - c*d through one Montgomery reduction (the y-coordinate of the XYZZ formulas), both signs of the difference."""
    mod = pyref.P_MOD
    rng = random.Random(5)
    edge = [0, 1, mod - 1, mod - 2, (1 << 253) % mod, (1 << 128) - 1]
    quads = [(a, b, c, d) for a in edge for b in edge for c in edge for d in edge] + [tuple(rng.randrange(mod) for _ in range(4)) for _ in range(5000)]
    cols = [orc.to_mont([q[i] for q in quads], mod) for i in range(4)]
    out = np.empty_like(cols[0])
    he.he_fq_mul_sub_mul(_p(out), _p(cols[0]), _p(cols[1]), _p(cols[2]), _p(cols[3]), ctypes.c_size_t(len(quads)))
    assert orc.from_mont(out, mod) == [(a * b - c * d) % mod for a, b, c, d in quads]


@pytest.mark.parametrize("field", ["fr", "fq"])
def test_field_ops_match_bigint(he, orc, field):
    mod = pyref.R_MOD if field == "fr" else pyref.P_MOD
    rng = random.Random(1234)
    a = _edge_and_random(mod, 400, rng)
    b = list(reversed(_edge_and_random(mod, 400, rng)))
    rng.shuffle(b)
    A = orc.to_mont(a, mod); B = orc.to_mont(b, mod)
    out = np.empty_like(A)
    n = ctypes.c_size_t(len(a))
    getattr(he, f"he_{field}_mul")(_p(out), _p(A), _p(B), n)
    assert orc.from_mont(out, mod) == [x * y % mod for x, y in zip(a, b)]
    getattr(he, f"he_{field}_add")(_p(out), _p(A), _p(B), n)
    assert orc.from_mont(out, mod) == [(x + y) % mod for x, y in zip(a, b)]
    getattr(he, f"he_{field}_sub")(_p(out), _p(A), _p(B), n)
    assert orc.from_mont(out, mod) == [(x - y) % mod for x, y in zip(a, b)]
    getattr(he, f"he_{field}_inv")(_p(out), _p(A), ctypes.c_size_t(40))
    assert orc.from_mont(out[:40], mod) == [pow(x, -1, mod) if x else 0 for x in a[:40]]


def test_fr_neg_and_from_mont(he, orc):
    rng = random.Random(7)
    a = _edge_and_random(pyref.R_MOD, 100, rng)
    A = orc.fr(a); out = np.empty_like(A)
    he.he_fr_neg(_p(out), _p(A), ctypes.c_size_t(len(a)))
    assert orc.fr_ints(out) == [(-x) % pyref.R_MOD for x in a]
    he.he_fr_from_mont(_p(out), _p(A), ctypes.c_size_t(len(a)))
    got = [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in out]
    assert got == a


def test_mul_worst_case_carries(he, orc):
    """operands with all-ones limbs below the modulus top: stresses every carry chain of the even/odd CIOS."""
    for mod, f in ((pyref.R_MOD, "fr"), (pyref.P_MOD, "fq")):
        vals = [mod - 1 - i for i in range(16)] + [((1 << 254) - 1) % mod, ((1 << 224) - 1), (mod >> 1), (mod >> 1) + 1]
        a = [x for x in vals for _ in vals]; b = [y for _ in vals for y in vals]
        # operands handed over WITHOUT Montgomery conversion: raw limb patterns are what matter here
        A = np.array([[(x >> (64 * j)) & (2**64 - 1) for j in range(4)] for x in a], dtype=np.uint64)
        B = np.array([[(x >> (64 * j)) & (2**64 - 1) for j in range(4)] for x in b], dtype=np.uint64)
        out = np.empty_like(A)
        getattr(he, f"he_{f}_mul")(_p(out), _p(A), _p(B), ctypes.c_size_t(len(a)))
        rinv = pow(1 << 256, -1, mod)
        got = [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in out]
        assert got == [x * y * rinv % mod for x, y in zip(a, b)]


def _rand_points(orc, n, seed):
    sc = orc.fr_random_chacha(n, seed)
    return orc.g1_fixed_base_mul(sc), orc.fr_ints(sc)


def test_curve_sums_match_python(he, orc):
    pts, ks = _rand_points(orc, 24, 99)
    want = pyref.ec_mul((1, 2), sum(ks) % pyref.R_MOD)
    for fn in ("he_sum_mixed", "he_sum_general"):
        out = np.empty(8, dtype=np.uint64)
        getattr(he, fn)(_p(out), _p(pts), ctypes.c_size_t(len(ks)))
        assert pyref.aff_tuple(orc.affine_ints(out)[0]) == want


def test_curve_exceptional_cases(he, orc):
    """P+P (doubling through the adder), P+(-P) (identity), identity operands, affine (0,0) entries."""
    g = orc.g1_generator()
    negg = g.copy(); negg[4:] = orc.fq([(-2) % pyref.P_MOD])[0]
    ident = np.zeros(8, dtype=np.uint64)
    cases = [
        ([g, g], pyref.ec_mul((1, 2), 2)),
        ([g, negg], None),
        ([ident, g, ident], (1, 2)),
        ([g, g, g, negg, g], pyref.ec_mul((1, 2), 3)),
        ([g, negg, g, g], pyref.ec_mul((1, 2), 2)),
        ([ident, ident], None),
    ]
    for pts, want in cases:
        arr = np.ascontiguousarray(np.stack(pts))
        for fn in ("he_sum_mixed", "he_sum_general"):
            out = np.empty(8, dtype=np.uint64)
            getattr(he, fn)(_p(out), _p(arr), ctypes.c_size_t(len(pts)))
            assert pyref.aff_tuple(orc.affine_ints(out)[0]) == want, (fn, want)


def test_small_scalar_mul_and_double(he, orc):
    g = orc.g1_generator()
    for k in (0, 1, 2, 3, 17, 65535, 65536, 0xFFFFFFFF):
        out = np.empty(8, dtype=np.uint64)
        he.he_mul_u32(_p(out), _p(g), ctypes.c_uint32(k))
        assert pyref.aff_tuple(orc.affine_ints(out)[0]) == pyref.ec_mul((1, 2), k)
    out = np.empty(8, dtype=np.uint64)
    he.he_dbl(_p(out), _p(g))
    assert orc.affine_ints(out)[0] == pyref.ec_mul((1, 2), 2)
    assert he.he_on_curve(_p(out)) == 1
    bad = out.copy(); bad[0] ^= np.uint64(1)
    assert he.he_on_curve(_p(bad)) == 0
    he.he_jac_roundtrip(_p(bad), _p(out))
    assert (bad == out).all()
