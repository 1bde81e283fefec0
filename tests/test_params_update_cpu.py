"""CPU tests of the params update chain in spectre_b200.plonk: the ParamsUpdate byte layout, the challenge's bytes, and
check_params_updates on the host stand-ins of tests/test_params_check_cpu.py (explicit params on the oracle's MSM, the
pure-Python pairing). The records are made by plonk.prove_params_update over the host backend, as contribute_params makes them
after the device update; the params a chain ends in are ParamsKZG::setup under the product of the secrets (secret_params)."""
import random

import numpy as np
import pytest

from spectre_b200 import halo2, plonk
from spectre_b200.transcript import keccak256
from tests import pypairing as pp
from tests import pyref
from tests.test_params_check_cpu import CheckedPairing, ExplicitEngine, corrupted, doubled, plus_generator, report, secret_params
from tests.verify_common import PyBackend

R = pp.R
K = 3


class CountingPairing(CheckedPairing):
    """CheckedPairing that also counts its pairing_check_batch calls"""

    def __init__(self):
        super().__init__()
        self.calls = 0

    def pairing_check_batch(self, ps, qs, m):
        self.calls += 1
        return super().pairing_check_batch(ps, qs, m)


def s_g2(s):
    return pp.g2_limbs(pp.g2_mul(pp.G2_GEN, s))


def start_vp(s0):
    return halo2.ParamsVerifierKZG(pp.g1_limbs(pp.G1_GEN), pp.g2_limbs(pp.G2_GEN), s_g2(s0))


def chain(s0, ts, rhos):
    """the records of updates by ts from the secret s0, and the secret they end in"""
    be, out, s = PyBackend(), [], s0
    for t, rho in zip(ts, rhos):
        out.append(plonk.prove_params_update(be, s_g2(s), s_g2(s * t % R), t, rho))
        s = s * t % R
    return out, s


@pytest.fixture(scope="module")
def setting(orc):
    rng = random.Random(0x9a7)
    s0 = rng.randrange(2, R)
    ts = [rng.randrange(2, R) for _ in range(3)]
    rhos = [rng.randrange(2, R) for _ in range(3)]
    updates, s = chain(s0, ts, rhos)
    return s0, ts, updates, secret_params(orc, K, s)


# ---- the record ---------------------------------------------------------------------------------------------------------
def test_record_bytes_round_trip_in_the_stated_layout():
    rng = random.Random(1)
    t, rho, s0 = (rng.randrange(2, R) for _ in range(3))
    u = plonk.prove_params_update(PyBackend(), s_g2(s0), s_g2(s0 * t % R), t, rho)
    raw = u.to_bytes()
    assert len(raw) == plonk.PARAMS_UPDATE_BYTES == 288
    assert raw[:128] == s_g2(s0 * t % R).tobytes()
    assert raw[128:192] == pp.g1_limbs(pyref.ec_mul(pp.G1_GEN, t)).tobytes()
    assert raw[192:256] == pp.g1_limbs(pyref.ec_mul(pp.G1_GEN, rho)).tobytes()
    assert raw[256:] == plonk.fr_mont(u.z).tobytes()
    back = plonk.ParamsUpdate.from_bytes(raw)
    assert back.to_bytes() == raw and back.z == u.z


def test_malformed_records_are_refused():
    u = plonk.prove_params_update(PyBackend(), s_g2(3), s_g2(6), 2, 5)
    raw = bytearray(u.to_bytes())
    with pytest.raises(ValueError, match="bytes"):
        plonk.ParamsUpdate.from_bytes(raw[:-1])
    for at, what in ((0, "s_g2"), (128, "T: x is not less"), (224, "R: y is not less")):
        bad = bytearray(raw); bad[at:at + 32] = (pp.P + 1).to_bytes(32, "little")
        with pytest.raises(ValueError, match=what):
            plonk.ParamsUpdate.from_bytes(bad)
    bad = bytearray(raw); bad[128:192] = pp.g1_limbs((1, 3)).tobytes()
    with pytest.raises(ValueError, match="T: not on the curve"):
        plonk.ParamsUpdate.from_bytes(bad)
    bad = bytearray(raw); bad[256:] = R.to_bytes(32, "little")
    with pytest.raises(ValueError, match="z is not less than r"):
        plonk.ParamsUpdate.from_bytes(bad)


def test_challenge_is_keccak_of_the_stated_concatenation():
    t, rho, s0 = 7, 11, 13
    u = plonk.prove_params_update(PyBackend(), s_g2(s0), s_g2(s0 * t), t, rho)
    fq = lambda vals: b"".join((v * (1 << 256) % pp.P).to_bytes(32, "little") for v in vals)
    before, after = pp.g2_mul(pp.G2_GEN, s0), pp.g2_mul(pp.G2_GEN, s0 * t)
    data = (b"spectre-b200 params update v1" + fq([before[0][0], before[0][1], before[1][0], before[1][1]])
            + fq([after[0][0], after[0][1], after[1][0], after[1][1]]) + fq(pyref.ec_mul(pp.G1_GEN, t)) + fq(pyref.ec_mul(pp.G1_GEN, rho)))
    c = int.from_bytes(keccak256(data), "big") % R
    assert plonk.params_update_challenge(s_g2(s0), u) == c
    assert u.z == (rho + c * t) % R


# ---- the chain ----------------------------------------------------------------------------------------------------------
def test_a_sound_chain_passes_with_one_pairing_call_for_its_ratios(setting):
    s0, _, updates, final = setting
    be = CountingPairing()
    assert plonk.check_params_updates(ExplicitEngine(final), be, start_vp(s0), updates, seed=b"\x01" * 32) == []
    assert be.calls == 2 and be.checks == 3 + 1                  # the ratios of three records, then check_params' chain check


def test_an_empty_chain_is_check_params_on_the_start(orc, setting):
    s0 = setting[0]
    own = secret_params(orc, K, s0)
    assert plonk.check_params_updates(ExplicitEngine(own), CheckedPairing(), start_vp(s0), [], seed=b"\x02" * 32) == []


def _cases(orc, setting):
    s0, ts, updates, final = setting
    u = list(updates)
    other_t = plonk.prove_params_update(PyBackend(), s_g2(s0 * ts[0] % R), updates[1].s_g2, 12345, 678)
    end = [("trailer", 1), ("powers", 1)]                      # final params whose own trailer is not the last record's s_g2
    return {
        "t_from_another_t": (u[:1] + [u[1]._replace(t_g1=other_t.t_g1)] + u[2:], final, [("ratio", 1)]),
        "t_from_another_t_reproved": (u[:1] + [other_t] + u[2:], final, [("ratio", 1)]),
        "changed_z": (u[:1] + [u[1]._replace(z=(u[1].z + 1) % R)] + u[2:], final, [("knowledge", 1)]),
        "s_g2_not_t_times_before": (u[:2] + [u[2]._replace(s_g2=pp.g2_limbs(pp.g2_add(pp.g2_from_limbs(u[2].s_g2), pp.G2_GEN)))], final,
                                    [("ratio", 2)] + end),
        "swapped": ([u[0], u[2], u[1]], final, [("ratio", 1), ("ratio", 2)] + end),
        "identity_t": ([u[0]._replace(t_g1=np.zeros(8, np.uint64))] + u[1:], final, [("degenerate", 0)]),
        "final_g_replaced": (u, corrupted(final, g=doubled(final.g, 5)), [("powers", 5), ("lagrange", 0)]),
        "final_g_lagrange_replaced": (u, corrupted(final, g_lagrange=plus_generator(final.g_lagrange, 6)), [("lagrange", 6)]),
    }


@pytest.mark.parametrize("name", ["t_from_another_t", "t_from_another_t_reproved", "changed_z", "s_g2_not_t_times_before", "swapped",
                                  "identity_t", "final_g_replaced", "final_g_lagrange_replaced"])
def test_each_failure_is_named(orc, setting, name):
    updates, final, want = _cases(orc, setting)[name]
    be = CountingPairing()
    got = plonk.check_params_updates(ExplicitEngine(final), be, start_vp(setting[0]), updates, seed=b"\x03" * 32)
    assert report(got) == want
    assert all(f.detail for f in got)
    assert isinstance(got[0], plonk.UpdateFailure) == (want[0][0] in ("degenerate", "ratio", "knowledge"))
