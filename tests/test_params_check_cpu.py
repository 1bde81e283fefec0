"""CPU tests of spectre_b200.plonk.check_params: the params check on the oracle's arithmetic, with a pure-Python pairing.

The oracle engine commits with the known-tau shortcut of the seed-0 SRS, which cannot represent corrupted params, so the engine
here commits with a real MSM (the oracle's best_multiexp) over the params' own bases, held on the host. The pairing is
tests/pypairing, refusing G2 inputs off the twist or outside the r-torsion subgroup as the library does. Small k keeps the
pure-Python pairings fast: a clean check costs one, a broken chain one more per bisection step."""
import random

import numpy as np
import pytest

from spectre_b200 import halo2, plonk
from tests import pypairing as pp
from tests import pyref
from tests.plonk_oracle_engine import OracleEngine
from tests.verify_common import PyBackend, contract_vp

G, GL = halo2.BASIS_G, halo2.BASIS_G_LAGRANGE


class HostParams:
    """the part of halo2.ParamsKZG that check_params reads, over host arrays; g_lagrange None is a from_bases handle"""

    def __init__(self, k, g, g_lagrange, trailer=None):
        self.k, self.n = k, 1 << k
        self.g = np.array(g, dtype=np.uint64).reshape(-1, 8)
        self.g_lagrange = None if g_lagrange is None else np.array(g_lagrange, dtype=np.uint64).reshape(-1, 8)
        self.g2, self.s_g2 = (np.zeros(16, np.uint64), np.zeros(16, np.uint64)) if trailer is None else [np.array(t, np.uint64).reshape(16) for t in trailer]

    def get_g(self, start=0, count=None, basis=G):
        src = self.g if basis == G else self.g_lagrange
        if src is None:
            raise halo2.BackendError("spb_srs_download: basis %d not resident" % basis)
        count = self.n - start if count is None else count
        return src[start:start + count].copy()

    def get_g2(self):
        return self.g2.copy(), self.s_g2.copy()

    def verifier_params(self):
        if not self.g2.any() or not self.s_g2.any():
            raise ValueError("verifier_params: the params hold no G2 points; set_g2 first")
        return halo2.ParamsVerifierKZG(self.g[0], self.g2, self.s_g2)


class ExplicitEngine(OracleEngine):
    """the oracle engine bound to explicit params: commit is best_multiexp over the params' first n bases"""

    def __init__(self, params, k=None):
        super().__init__(params.k if k is None else k, 3)
        self.params = params

    def zero(self, b):
        b.a[:] = 0

    def commit(self, basis, bufs, n):
        from oracle import oracle as orc
        bases = self.params.get_g(0, n, basis)
        return [halo2.jacobian_to_affine_ints(orc.best_multiexp(np.ascontiguousarray(b.a[:n]), bases)) for b in bufs]


class CheckedPairing(PyBackend):
    """PyBackend whose pairing refuses a G2 input off the twist or outside the r-torsion subgroup with the library's error text,
    and counts its checks"""

    def __init__(self):
        self.checks = 0

    def pairing_check_batch(self, ps, qs, m):
        for i, q in enumerate(np.asarray(qs, dtype=np.uint64).reshape(-1, 16)):
            pt = pp.g2_from_limbs(q)
            why = "not on the curve" if not pp.g2_on_curve(pt) else "not in the r-torsion subgroup" if pp.g2_mul(pt, pp.R) is not None else None
            if why:
                raise halo2.BackendError("spb_pairing_check_batch failed (%d): spb_pairing_check_batch: q[%d]: %s" % (halo2.ERR_DATA, i, why))
        out = super().pairing_check_batch(ps, qs, m)
        self.checks += len(out)
        return out


# ---- params -----------------------------------------------------------------------------------------------------------
def seed0_params(orc, k, trailer=True):
    """the seed-0 SRS of the oracle (the one the verifier contracts carry -[s]_2 of), with its G2 trailer"""
    n = 1 << k
    tr = (pp.g2_limbs(pp.G2_GEN), orc.srs_s_g2().reshape(16)) if trailer else None
    return HostParams(k, orc.srs_g(k, 0, n), orc.srs_g_lagrange(k, 0, n), tr)


def secret_params(orc, k, s, trailer=True):
    """ParamsKZG::setup under the secret s: g[i] = s^i G, g_lagrange[i] = L_i(s) G, trailer ([1]_2, [s]_2)"""
    n, R = 1 << k, pp.R
    w = pyref.omega(k)
    lag = [pow(w, i, R) * (pow(s, n, R) - 1) * pow(n * (s - pow(w, i, R)), -1, R) % R for i in range(n)]
    g = orc.g1_fixed_base_mul(plonk.fr_mont_rows([pow(s, i, R) for i in range(n)]))
    gl = orc.g1_fixed_base_mul(plonk.fr_mont_rows(lag))
    tr = (pp.g2_limbs(pp.G2_GEN), pp.g2_limbs(pp.g2_mul(pp.G2_GEN, s))) if trailer else None
    return HostParams(k, g, gl, tr)


def point(limbs):
    return pyref.aff_tuple(tuple(pp.fq_ints(limbs)))


def doubled(bases, i):
    """bases with row i replaced by twice itself"""
    out = np.array(bases, dtype=np.uint64).copy()
    p = point(out[i])
    out[i] = pp.g1_limbs(pyref.ec_add(p, p))
    return out


def plus_generator(bases, i):
    """bases with row i replaced by itself + G"""
    out = np.array(bases, dtype=np.uint64).copy()
    out[i] = pp.g1_limbs(pyref.ec_add(point(out[i]), pp.G1_GEN))
    return out


def swapped(bases, a, b):
    out = np.array(bases, dtype=np.uint64).copy()
    out[[a, b]] = out[[b, a]]
    return out


def corrupted(params, g=None, g_lagrange=None):
    return HostParams(params.k, params.g if g is None else g, params.g_lagrange if g_lagrange is None else g_lagrange, (params.g2, params.s_g2))


def corruption_cases(orc, k):
    """(name, params, the expected report against the contract vp as (kind, index) pairs) on the seed-0 SRS at k"""
    n = 1 << k
    base = seed0_params(orc, k)
    g, gl = base.g, base.g_lagrange
    cases = [("clean", base, [])]
    for j in (1, n // 2, n - 1):
        cases.append(("g%d_doubled" % j, corrupted(base, g=doubled(g, j)), [("powers", j), ("lagrange", 0)]))
    for i in (0, n - 1):
        cases.append(("gl%d_plus_G" % i, corrupted(base, g_lagrange=plus_generator(gl, i)), [("lagrange", i)]))
    cases.append(("gl_swapped", corrupted(base, g_lagrange=swapped(gl, 2, n - 3)), [("lagrange", 2)]))
    cases.append(("both", corrupted(base, g=doubled(g, n // 2), g_lagrange=plus_generator(gl, 1)), [("powers", n // 2), ("lagrange", 0)]))
    two_g = pp.g1_limbs(pyref.ec_add(pp.G1_GEN, pp.G1_GEN))
    g0 = g.copy(); g0[0] = two_g
    cases.append(("g0_is_2G", corrupted(base, g=g0), [("g_generator", 0), ("powers", 1), ("lagrange", 0)]))
    return cases


def report(got):
    return [(f.kind, f.index) for f in got]


# ---- tests ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [3, 5])
def test_seed0_params_pass_against_the_contract_and_their_own_trailer(orc, kats, k):
    params = seed0_params(orc, k)
    be = CheckedPairing()
    assert plonk.check_params(ExplicitEngine(params), be, contract_vp(kats), seed=b"\x01" * 32) == []
    assert be.checks == 1
    timings = {}
    assert plonk.check_params(ExplicitEngine(params), be, seed=b"\x02" * 32, timings=timings) == []
    assert set(timings) == {"points", "powers", "lagrange"}


def test_params_under_another_secret(orc, kats):
    s = random.Random(7).randrange(2, pp.R)
    own = secret_params(orc, 3, s)
    be = CheckedPairing()
    assert plonk.check_params(ExplicitEngine(own), be, seed=b"\x03" * 32) == []
    assert report(plonk.check_params(ExplicitEngine(own), be, contract_vp(kats), seed=b"\x04" * 32)) == [("trailer", 1), ("powers", 1)]
    bare = secret_params(orc, 3, s, trailer=False)
    assert report(plonk.check_params(ExplicitEngine(bare), be, contract_vp(kats), seed=b"\x05" * 32)) == [("powers", 1)]


@pytest.mark.parametrize("name", ["clean", "g1_doubled", "g4_doubled", "g7_doubled", "gl0_plus_G", "gl7_plus_G", "gl_swapped", "both", "g0_is_2G"])
def test_corrupted_points_are_named(orc, kats, name):
    params, want = {c[0]: c[1:] for c in corruption_cases(orc, 3)}[name]
    be = CheckedPairing()
    got = plonk.check_params(ExplicitEngine(params), be, contract_vp(kats), seed=b"\x06" * 32)
    assert report(got) == want
    assert all(f.detail for f in got)
    # one check over the whole chain, then at most ceil(log2(n - 1)) = 3 bisection steps when it breaks
    assert 1 < be.checks <= 4 if "powers" in dict(want) else be.checks == 1


def test_s_g2_outside_the_subgroup_is_named(orc, kats):
    outside = pp.g2_twist_point_outside_subgroup()
    vp = contract_vp(kats, s_g2=outside)
    bare = seed0_params(orc, 3, trailer=False)
    got = plonk.check_params(ExplicitEngine(bare), CheckedPairing(), vp, seed=b"\x07" * 32)
    assert report(got) == [("s_g2", 0)] and "not in the r-torsion subgroup" in got[0].detail
    got = plonk.check_params(ExplicitEngine(seed0_params(orc, 3)), CheckedPairing(), vp, seed=b"\x07" * 32)
    assert report(got) == [("trailer", 1), ("s_g2", 0)]


def test_a_wrong_g2_generator_is_named(orc, kats):
    vp = contract_vp(kats)
    vp.g2 = pp.g2_limbs(pp.g2_add(pp.G2_GEN, pp.G2_GEN))
    got = plonk.check_params(ExplicitEngine(seed0_params(orc, 3, trailer=False)), CheckedPairing(), vp, seed=b"\x08" * 32)
    assert report(got) == [("g2_generator", 0), ("powers", 1)]


def test_the_same_seed_gives_the_same_report_and_other_seeds_catch_the_point(orc, kats):
    base = seed0_params(orc, 3)
    params = corrupted(base, g=doubled(base.g, 5), g_lagrange=plus_generator(base.g_lagrange, 6))
    vp = contract_vp(kats)
    first = plonk.check_params(ExplicitEngine(params), CheckedPairing(), vp, seed=b"\x09" * 32)
    assert plonk.check_params(ExplicitEngine(params), CheckedPairing(), vp, seed=b"\x09" * 32) == first
    one_bad = corrupted(base, g_lagrange=plus_generator(base.g_lagrange, 3))
    for seed in (b"\x0a" * 32, bytes(range(32)), None):
        assert report(plonk.check_params(ExplicitEngine(one_bad), CheckedPairing(), vp, seed=seed)) == [("lagrange", 3)]


def test_handles_that_are_not_checked_params_are_refused(orc, kats):
    params = seed0_params(orc, 3)
    with pytest.raises(ValueError, match="from_bases"):
        plonk.check_params(ExplicitEngine(HostParams(3, params.g, None)), CheckedPairing(), contract_vp(kats))
    with pytest.raises(ValueError, match="engine is for k = 4"):
        plonk.check_params(ExplicitEngine(params, k=4), CheckedPairing(), contract_vp(kats))
    with pytest.raises(ValueError, match="set_g2 first"):
        plonk.check_params(ExplicitEngine(seed0_params(orc, 3, trailer=False)), CheckedPairing())
