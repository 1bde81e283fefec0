"""CPU-only tests of the pairing's device bodies (spectre_b200/csrc/pairing.cuh) against the pure-Python reference
(tests/pypairing.py), which shares only the tower with them.

tests/hostemu/pairing.cpp is compiled for the host with -DSPB_EMULATE_PTX (the 32-bit-limb carry chains the GPU runs) and
without it (the 64-bit host path the library's error text takes). Covered: Fq6 and Fq12 mul, sqr and inverse, the sparse line
product, the three Frobenius maps, the Miller loop followed by the final exponentiation, identity pairs, and the G2 check
(a multiple of the generator passes; a twist point outside the order-r subgroup, found without clearing the cofactor, fails).
"""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import pypairing as pp
from tests import pyref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu")
P = pp.P


@pytest.fixture(scope="module", params=["ptx", "native"])
def he(request, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostemu_pairing") / ("libhostemu_%s.so" % request.param))
    flags = ["-DSPB_EMULATE_PTX"] if request.param == "ptx" else []
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-o", so, os.path.join(HERE, "pairing.cpp")])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def rand_f6(rng):
    return pp.f6_unflat([rng.randrange(P) for _ in range(6)])


def rand_f12(rng):
    return pp.f12_unflat([rng.randrange(P) for _ in range(12)])


def f6_limbs(xs):
    return np.concatenate([pp.fq_limbs(pp.f6_flat(x)) for x in xs]) if xs else np.zeros((0, 4), np.uint64)


def f12_limbs(xs):
    return np.concatenate([pp.gt_limbs(x) for x in xs])


def run6(he, op, a, b=None):
    A = f6_limbs(a)
    B = f6_limbs(b) if b is not None else np.zeros_like(A)
    out = np.empty_like(A)
    he.he_fq6_op(op, _p(A), _p(B), _p(out), ctypes.c_size_t(len(a)))
    v = pp.fq_ints(out)
    return [pp.f6_unflat(v[6 * i:6 * i + 6]) for i in range(len(a))]


def run12(he, op, a, b=None):
    A = f12_limbs(a)
    B = f12_limbs(b) if b is not None else np.zeros_like(A)
    out = np.empty_like(A)
    he.he_fq12_op(op, _p(A), _p(B), _p(out), ctypes.c_size_t(len(a)))
    v = pp.fq_ints(out)
    return [pp.f12_unflat(v[12 * i:12 * i + 12]) for i in range(len(a))]


def he_pairing(he, ps, qs):
    P_ = np.stack([pp.g1_limbs(p) for p in ps]) if ps else np.zeros((0, 8), np.uint64)
    Q_ = np.stack([pp.g2_limbs(q) for q in qs]) if qs else np.zeros((0, 16), np.uint64)
    out = np.empty((12, 4), np.uint64)
    he.he_pairing(_p(P_), _p(Q_), ctypes.c_size_t(len(ps)), _p(out))
    return pp.gt_from_limbs(out)


def test_fq6_mul_sqr_inv(he):
    rng = random.Random(61)
    a = [rand_f6(rng) for _ in range(12)] + [pp.F6_ONE, ((P - 1, P - 1), (P - 1, 0), (0, P - 1))]
    b = [rand_f6(rng) for _ in range(len(a))]
    assert run6(he, 0, a, b) == [pp.f6_mul(x, y) for x, y in zip(a, b)]
    assert run6(he, 1, a) == [pp.f6_mul(x, x) for x in a]
    inv = run6(he, 2, a)
    assert inv == [pp.f6_inv(x) for x in a]
    assert all(pp.f6_mul(x, y) == pp.F6_ONE for x, y in zip(a, inv))


def test_fq12_mul_sqr_inv_and_sparse_line(he):
    rng = random.Random(62)
    a = [rand_f12(rng) for _ in range(8)] + [pp.F12_ONE]
    b = [rand_f12(rng) for _ in range(len(a))]
    assert run12(he, 0, a, b) == [pp.f12_mul(x, y) for x, y in zip(a, b)]
    assert run12(he, 1, a) == [pp.f12_sqr(x) for x in a]
    inv = run12(he, 2, a)
    assert inv == [pp.f12_inv(x) for x in a]
    assert all(pp.f12_mul(x, y) == pp.F12_ONE for x, y in zip(a, inv))
    # a line has three non-zero coefficients: w^0 (c0.c0), w^1 (c1.c0), w^3 (c1.c1)
    lines = [((l[0][0], pp.F2_ZERO, pp.F2_ZERO), (l[1][0], l[1][1], pp.F2_ZERO)) for l in b]
    assert run12(he, 6, a, lines) == [pp.f12_mul(x, l) for x, l in zip(a, lines)]


@pytest.mark.parametrize("k", [1, 2, 3])
def test_fq12_frobenius_maps(he, k):
    rng = random.Random(63 + k)
    a = [rand_f12(rng) for _ in range(3)]
    assert run12(he, 2 + k, a) == [pp.f12_frobenius(x, k) for x in a]


def test_miller_loop_and_final_exponentiation_give_the_reference_gt(he):
    rng = random.Random(64)
    for _ in range(2):
        a, b = rng.randrange(1, pp.R), rng.randrange(1, pp.R)
        p, q = pyref.ec_mul(pp.G1_GEN, a), pp.g2_mul(pp.G2_GEN, b)
        assert he_pairing(he, [p], [q]) == pp.pairing(p, q)
    # a product of two pairs under one final exponentiation, and a balanced check
    a = rng.randrange(1, pp.R)
    p1, q1 = pyref.ec_mul(pp.G1_GEN, a), pp.G2_GEN
    p2, q2 = pyref.ec_mul(pp.G1_GEN, pp.R - 1), pp.g2_mul(pp.G2_GEN, a)
    assert he_pairing(he, [p1, p2], [q1, pp.G2_GEN]) == pp.multi_pairing([p1, p2], [q1, pp.G2_GEN])
    assert he_pairing(he, [p1, p2], [q1, q2]) == pp.F12_ONE


def test_identity_pairs_contribute_one(he):
    g = pp.pairing(pp.G1_GEN, pp.G2_GEN)
    assert he_pairing(he, [None], [pp.G2_GEN]) == pp.F12_ONE
    assert he_pairing(he, [pp.G1_GEN], [None]) == pp.F12_ONE
    assert he_pairing(he, [None, pp.G1_GEN, pp.G1_GEN], [None, pp.G2_GEN, None]) == g
    assert he_pairing(he, [], []) == pp.F12_ONE


def test_g2_subgroup_check(he):
    rng = random.Random(65)
    inside = [pp.G2_GEN, pp.g2_mul(pp.G2_GEN, rng.randrange(1, pp.R)), pp.g2_mul(pp.G2_GEN, pp.R - 1), None]
    outside = pp.g2_twist_point_outside_subgroup()
    assert pp.g2_on_curve(outside) and pp.g2_mul(outside, pp.R) is not None
    off = (pp.G2_GEN[0], pp.f2_add(pp.G2_GEN[1], (1, 0)))
    pts = inside + [outside, pp.g2_neg(outside), off]
    Q = np.stack([pp.g2_limbs(q) for q in pts])
    big = Q[0].copy(); big[0:4] = np.array([(P >> (64 * j)) & ((1 << 64) - 1) for j in range(4)], np.uint64)   # x.c0 = p, raw
    Q = np.concatenate([Q, big[None]])
    out = np.empty(Q.shape[0], np.int32)
    he.he_g2_pairing_check(_p(out), _p(Q), ctypes.c_size_t(Q.shape[0]))
    assert out.tolist() == [0, 0, 0, 0, 4, 4, 3, 1]
