"""The BN254 pairing on the GPU (spb_pairing, spb_pairing_check_batch) against the pure-Python reference tests/pypairing.py."""
import ctypes
import random

import numpy as np
import pytest

from spectre_b200 import halo2
from tests import pypairing as pp
from tests import pyref
from tests.gpu_common import be, device_lists  # noqa: F401

pytestmark = pytest.mark.gpu


def _g1(points):
    return np.stack([pp.g1_limbs(p) for p in points])


def _g2(points):
    return np.stack([pp.g2_limbs(q) for q in points])


def _random_pairs(seed, n):
    rng = random.Random(seed)
    return ([pyref.ec_mul(pp.G1_GEN, rng.randrange(1, pp.R)) for _ in range(n)],
            [pp.g2_mul(pp.G2_GEN, rng.randrange(1, pp.R)) for _ in range(n)])


def test_pairing_matches_the_reference_on_random_pairs(be):
    ps, qs = _random_pairs(81, 8)
    for p, q in zip(ps, qs):
        assert pp.gt_from_limbs(be.pairing(_g1([p]), _g2([q]))) == pp.pairing(p, q)
    assert pp.gt_from_limbs(be.pairing(_g1(ps), _g2(qs))) == pp.multi_pairing(ps, qs)


def test_pairing_is_bilinear(be):
    rng = random.Random(82)
    a, b = rng.randrange(1, pp.R), rng.randrange(1, pp.R)
    e = pp.gt_from_limbs(be.pairing(_g1([pp.G1_GEN]), _g2([pp.G2_GEN])))
    eab = pp.gt_from_limbs(be.pairing(_g1([pyref.ec_mul(pp.G1_GEN, a)]), _g2([pp.g2_mul(pp.G2_GEN, b)])))
    assert e != pp.F12_ONE and eab == pp.f12_pow(e, a * b % pp.R)


def test_identity_pairs_and_the_empty_product_give_one(be):
    one = pp.F12_ONE
    assert pp.gt_from_limbs(be.pairing(_g1([None, pp.G1_GEN]), _g2([pp.G2_GEN, None]))) == one
    assert pp.gt_from_limbs(be.pairing(np.zeros((0, 8), np.uint64), np.zeros((0, 16), np.uint64))) == one
    assert be.pairing_check_batch(_g1([None, None]), _g2([None, pp.G2_GEN]), 2) == [True]


@pytest.mark.parametrize("ids", device_lists())
def test_same_result_on_a_context_of_several_device_entries(be, ids):
    ps, qs = _random_pairs(83, 3)
    want = be.pairing(_g1(ps), _g2(qs))
    be2 = halo2.Backend(ids)
    try:
        assert np.array_equal(be2.pairing(_g1(ps), _g2(qs)), want)
        assert be2.pairing_check_batch(_g1(ps[:2]), _g2(qs[:2]), 1) == [False, False]
    finally:
        be2.close()


def _check_pool():
    """balanced checks e(aP, Q) e(-P, aQ) = 1 and unbalanced ones e(aP, Q) e(-P, (a + 1)Q) != 1, a few distinct of each"""
    rng = random.Random(84)
    pool = []
    for i in range(6):
        a = rng.randrange(2, pp.R)
        p, q = pyref.ec_mul(pp.G1_GEN, rng.randrange(1, pp.R)), pp.g2_mul(pp.G2_GEN, rng.randrange(1, pp.R))
        ap, aq = pyref.ec_mul(p, a), pp.g2_mul(q, a)
        neg_p = (p[0], (-p[1]) % pp.P)
        if i % 2 == 0:
            pool.append(((ap, neg_p), (q, aq), True))
        else:
            pool.append(((ap, neg_p), (q, pp.g2_add(aq, q)), False))
    return pool


@pytest.mark.parametrize("n_checks", [1, 7, 1000, 8192])
def test_check_batch_returns_the_verdict_of_every_check(be, n_checks):
    pool = _check_pool()
    g1 = [_g1(ps) for ps, _, _ in pool]
    g2 = [_g2(qs) for _, qs, _ in pool]
    pick = [(j * 7 + j // 5) % len(pool) for j in range(n_checks)]
    ps = np.concatenate([g1[i] for i in pick])
    qs = np.concatenate([g2[i] for i in pick])
    before = be.kernel_launches
    got = be.pairing_check_batch(ps, qs, 2)
    assert be.kernel_launches - before == 3
    assert got == [pool[i][2] for i in pick]
    assert be.last_device_ms > 0


def _raw(be, ps, qs, m):
    """spb_pairing_check_batch through ctypes: (rc, error text, the ok array as the call left it)"""
    ok = np.full(ps.shape[0] // m, 7, dtype=np.int32)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = be.lib.spb_pairing_check_batch(be.ctx, vp(ps), vp(qs), ctypes.c_size_t(m), ctypes.c_size_t(ps.shape[0] // m), vp(ok))
    return rc, be.lib.spb_last_error(be.ctx).decode(), ok


def test_invalid_inputs_are_named_and_leave_the_output_untouched(be):
    ps, qs = _random_pairs(85, 8)
    P_, Q_ = _g1(ps), _g2(qs)
    p_big = P_.copy(); p_big[3, 0:4] = np.array([(pp.P >> (64 * j)) & ((1 << 64) - 1) for j in range(4)], np.uint64)
    p_off = P_.copy(); p_off[5] = pp.g1_limbs((ps[5][0], (ps[5][1] + 1) % pp.P))
    q_off = Q_.copy(); q_off[6] = pp.g2_limbs((qs[6][0], pp.f2_add(qs[6][1], (1, 0))))
    q_sub = Q_.copy(); q_sub[2] = pp.g2_limbs(pp.g2_twist_point_outside_subgroup())
    cases = [(p_big, Q_, "p[3]: x is not less than the field modulus"), (P_, q_off, "q[6]: not on the curve"),
             (p_off, Q_, "p[5]: not on the curve"), (P_, q_sub, "q[2]: not in the r-torsion subgroup")]
    for ps_, qs_, text in cases:
        rc, err, ok = _raw(be, ps_, qs_, 2)
        assert rc == halo2.ERR_DATA and text in err and (ok == 7).all(), (text, err)
    # the first invalid input in the order p[0], q[0], p[1], q[1], ...
    rc, err, _ = _raw(be, p_off, q_sub, 2)
    assert rc == halo2.ERR_DATA and "q[2]: not in the r-torsion subgroup" in err
    with pytest.raises(halo2.BackendError, match="not on the curve"):
        be.pairing(p_off, Q_)
