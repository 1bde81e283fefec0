"""CPU-only tests of the params-file point checks (spectre_b200/csrc/{field,curve}.cuh: fp_is_canonical, affine_check,
g2_affine_check), the predicates the checked ParamsKZG read runs on the device and on the host.

tests/hostemu/srs_check.cpp is compiled for the host with -DSPB_EMULATE_PTX (the 32-bit-limb carry chains the GPU runs) and
without it (the 64-bit host path the library's G2 trailer check takes). Every verdict is compared with a Python big-integer
restatement: 0 valid, 1 x not less than p, 2 y not less than p, 3 off the curve. The G2 twist constant b' = 3 / (9 + u) is
derived here on its own, so the oracle's g2 and s_g2 passing cross-checks the constant compiled into the library.
"""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import pyref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu")
P = pyref.P_MOD
MONT_R = 1 << 256
RINV = pow(MONT_R, -1, P)
M64 = (1 << 64) - 1


@pytest.fixture(scope="module", params=["ptx", "native"])
def he(request, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostemu_srs") / ("libhostemu_%s.so" % request.param))
    flags = ["-DSPB_EMULATE_PTX"] if request.param == "ptx" else []
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, os.path.join(HERE, "srs_check.cpp")])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def ints_to_limbs(vals):
    """raw 256-bit integers (stored limbs, no Montgomery conversion) -> (n, 4) uint64"""
    return np.array([[(v >> (64 * j)) & M64 for j in range(4)] for v in vals], dtype=np.uint64).reshape(-1, 4)


def limbs_to_ints(arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 4)
    return [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in arr]


def mont(v):
    return v % P * MONT_R % P


# ---- Python restatement ----------------------------------------------------------------------------------------------
def g1_verdict(xr, yr):
    if xr >= P:
        return 1
    if yr >= P:
        return 2
    if xr == 0 and yr == 0:
        return 0
    x, y = xr * RINV % P, yr * RINV % P
    return 0 if (y * y - x * x * x - 3) % P == 0 else 3


def f2_mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def f2_inv(a):
    d = pow(a[0] * a[0] + a[1] * a[1], -1, P)
    return (a[0] * d % P, -a[1] * d % P)


B_TWIST = f2_mul((3, 0), f2_inv((9, 1)))       # b' = 3 / (9 + u) in Fq[u]/(u^2 + 1)


def g2_verdict(c):
    """c = stored limbs of (x.c0, x.c1, y.c0, y.c1) as ints"""
    if c[0] >= P or c[1] >= P:
        return 1
    if c[2] >= P or c[3] >= P:
        return 2
    if not any(c):
        return 0
    x = (c[0] * RINV % P, c[1] * RINV % P)
    y = (c[2] * RINV % P, c[3] * RINV % P)
    rhs = f2_mul(f2_mul(x, x), x)
    rhs = ((rhs[0] + B_TWIST[0]) % P, (rhs[1] + B_TWIST[1]) % P)
    return 0 if f2_mul(y, y) == rhs else 3


def run_g1(he, pairs):
    arr = np.ascontiguousarray(np.concatenate([ints_to_limbs([x for x, _ in pairs]), ints_to_limbs([y for _, y in pairs])], axis=1))
    out = np.empty(len(pairs), dtype=np.int32)
    he.he_g1_check(_p(out), _p(arr), ctypes.c_size_t(len(pairs)))
    return [int(v) for v in out]


def run_g2(he, quads):
    arr = np.ascontiguousarray(ints_to_limbs([v for q in quads for v in q]).reshape(-1, 16))
    out = np.empty(len(quads), dtype=np.int32)
    he.he_g2_check(_p(out), _p(arr), ctypes.c_size_t(len(quads)))
    return [int(v) for v in out]


def oracle_points(orc, k=6):
    pts = np.concatenate([orc.srs_g(k, 0, 1 << k), orc.srs_g_lagrange(k, 0, 1 << k)])
    xs, ys = limbs_to_ints(pts[:, :4]), limbs_to_ints(pts[:, 4:])
    return list(zip(xs, ys))


def oracle_g2(orc):
    g2 = np.empty((4, 4), dtype=np.uint64); s_g2 = np.empty((4, 4), dtype=np.uint64)
    orc.lib().orc_srs_g2_raw(_p(g2), _p(s_g2))
    return [tuple(limbs_to_ints(g2)), tuple(limbs_to_ints(s_g2))]


def test_twist_constant_is_three_over_nine_plus_u():
    assert f2_mul(B_TWIST, (9, 1)) == (3, 0)


def test_g1_valid_points_and_identity(he, orc):
    pts = oracle_points(orc)
    neg = [(x, (P - y) % P) for x, y in pts]                       # -P is on the curve too
    cases = pts + neg + [(0, 0)]
    assert [g1_verdict(x, y) for x, y in cases] == [0] * len(cases)
    assert run_g1(he, cases) == [0] * len(cases)


def test_g1_points_that_cannot_exist(he, orc):
    """(0, y): 3 is not a square mod p, so no point has x = 0. (x, 0): -3 is not a cube mod p, so no point has y = 0."""
    assert pow(3, (P - 1) // 2, P) == P - 1
    assert (P - 1) % 3 == 0 and pow(P - 3, (P - 1) // 3, P) != 1
    xs = [x for x, _ in oracle_points(orc)]
    cases = [(0, mont(1)), (0, 1), (0, mont(2))] + [(x, 0) for x in xs]
    want = [g1_verdict(x, y) for x, y in cases]
    assert want == [3] * len(cases)
    assert run_g1(he, cases) == want


def test_g1_coordinates_plus_multiples_of_p_are_not_canonical(he, orc):
    """x + j p and y + j p (j = 1..4) stay below 2^256 and are on the curve mod p, but the stored limbs are not reduced."""
    pts = oracle_points(orc)[:16]
    cases, want = [], []
    for x, y in pts:
        for j in range(1, 5):
            assert x + j * P < MONT_R and y + j * P < MONT_R
            cases += [(x + j * P, y), (x, y + j * P), (x + j * P, y + j * P)]
            want += [1, 2, 1]
    cases += [(P, 0), (0, P), (P - 1, P), (MONT_R - 1, MONT_R - 1), (pts[0][0], MONT_R - 1), (MONT_R - 1, pts[0][1])]
    want += [1, 2, 2, 1, 2, 1]
    assert [g1_verdict(x, y) for x, y in cases] == want
    assert run_g1(he, cases) == want


def test_g1_single_bit_flips(he, orc):
    pts = oracle_points(orc)
    rng = random.Random(3)
    cases = []
    for x, y in rng.sample(pts, 8) + [(0, 0)]:
        for b in range(256):
            cases += [(x ^ (1 << b), y), (x, y ^ (1 << b))]
    want = [g1_verdict(x, y) for x, y in cases]
    assert 0 not in want and {1, 2, 3} <= set(want)
    assert run_g1(he, cases) == want


def test_g1_random_limbs(he):
    rng = random.Random(11)
    cases = [(rng.getrandbits(256), rng.getrandbits(256)) for _ in range(3000)]
    cases += [(rng.randrange(P), rng.randrange(P)) for _ in range(2000)]
    # limbs equal to p's above a random limb, to reach every position of the top-down comparison
    for _ in range(500):
        i = rng.randrange(4)
        hi = P >> (64 * i) << (64 * i)
        cases.append((hi | rng.getrandbits(64 * i) if i else hi | rng.getrandbits(1), rng.randrange(P)))
    want = [g1_verdict(x, y) for x, y in cases]
    assert {1, 2, 3} <= set(want)
    assert run_g1(he, cases) == want


def test_g2_oracle_trailer_and_identity(he, orc):
    g2, s_g2 = oracle_g2(orc)
    neg = (g2[0], g2[1], (P - g2[2]) % P, (P - g2[3]) % P)
    cases = [g2, s_g2, neg, (0, 0, 0, 0)]
    assert [g2_verdict(c) for c in cases] == [0, 0, 0, 0]
    assert run_g2(he, cases) == [0, 0, 0, 0]


def test_g2_bit_flips_and_non_canonical_components(he, orc):
    cases = []
    for q in oracle_g2(orc):
        for c in range(4):
            for b in range(256):
                t = list(q); t[c] ^= 1 << b; cases.append(tuple(t))
            for j in range(1, 5):
                t = list(q); t[c] += j * P; cases.append(tuple(t))
            t = list(q); t[c] = P; cases.append(tuple(t))
    cases += [(0, 0, 0, mont(1)), (0, 0, mont(1), 0), (mont(1), 0, 0, 0), (MONT_R - 1,) * 4]
    want = [g2_verdict(c) for c in cases]
    assert 0 not in want and {1, 2, 3} <= set(want)
    assert run_g2(he, cases) == want
