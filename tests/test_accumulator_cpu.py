"""CPU-only tests of the KZG accumulator of an aggregation proof (spectre_b200.plonk: accumulator_to_limbs /
accumulator_from_limbs, succinct_verify, aggregate_accumulators, evm_pairing_points and verify_proof's accumulator_indices),
with the pure-Python stand-in for the device calls (tests/verify_common.PyBackend).

The limb decoder is held to the verifier contract's own rules. On the committed fixtures the decoded accumulator, r and the
two points the contract pairs are among the words the contract stored while accepting them, and on the three K = 23 proofs of
tests/golden/accumulator_contract_runs.json the accumulator check gives the contract's verdicts, where the check without
indices accepts all three. A two-layer run on the oracle engine carries an inner snark's accumulator into an outer proof."""
import json
import os
import random

import pytest

from spectre_b200 import circuits, halo2, plonk, poseidon
from spectre_b200.transcript import EvmTranscriptWrite
from tests import pypairing as pp
from tests import pyref
from tests.plonk_oracle_engine import OracleEngine, SeededRng
from tests.verify_common import GOLDEN, PyBackend, contract_g2, contract_vp, fixtures, load_fixture
from tools import make_k23_fixture

BE = PyBackend()
IDX = plonk.AGGREGATION_ACCUMULATOR_INDICES
G1 = (1, 2)


def _tau(orc):
    return orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]


def _limbs(v):
    return [v & ((1 << 88) - 1), (v >> 88) & ((1 << 88) - 1), v >> 176]


def _words(lhs, rhs):
    return _limbs(lhs[0]) + _limbs(lhs[1]) + _limbs(rhs[0]) + _limbs(rhs[1])


def _acc(rng, tau, good=True):
    rhs = pyref.ec_mul(G1, rng.randrange(1, pp.R))
    return plonk.KzgAccumulator(pyref.ec_mul(rhs, tau if good else tau + 1), rhs)


# ---- the limb codec ---------------------------------------------------------------------------------------------------
def test_limbs_round_trip_random_points():
    rng = random.Random(1)
    for _ in range(8):
        acc = plonk.KzgAccumulator(pyref.ec_mul(G1, rng.randrange(1, pp.R)), pyref.ec_mul(G1, rng.randrange(1, pp.R)))
        words = plonk.accumulator_to_limbs(acc)
        assert len(words) == 12 and all(0 <= w < 1 << 88 for w in words)
        assert words == _words(acc.lhs, acc.rhs)
        assert plonk.accumulator_from_limbs(words) == acc
    assert plonk.AGGREGATION_ACCUMULATOR_INDICES == [(0, i) for i in range(12)]


def test_limb_decoding_mirrors_the_contract():
    rng = random.Random(2)
    lhs, rhs = pyref.ec_mul(G1, rng.randrange(1, pp.R)), pyref.ec_mul(G1, rng.randrange(1, pp.R))
    acc = plonk.KzgAccumulator(lhs, rhs)
    w = _words(lhs, rhs)
    dec = plonk.accumulator_from_limbs

    def with_x(x):                                              # lhs.x limbs replaced, nothing else
        return _limbs(x) + w[3:]
    # every word is reduced mod r first
    assert dec([v + pp.R if i in (0, 4, 11) else v for i, v in enumerate(w)]) == acc
    # limbs of 88 bits or more overlap: l0 + 2^88 with l1 - 1 is the same coordinate
    ov = list(w)
    if ov[1] == 0:
        ov[1], ov[2] = (1 << 88), ov[2] - 1
    ov[0], ov[1] = ov[0] + (1 << 88), ov[1] - 1
    assert dec(ov) == acc
    # the top limb is shifted left by 176 with the EVM's wrap-around mod 2^256: a limb 2^80 more is the same coordinate,
    # where an exact decoder would see x + 2^256 >= p
    assert dec(w[:2] + [w[2] + (1 << 80)] + w[3:]) == acc
    # x or y >= p is refused even though it is the same point mod p
    assert dec(with_x(lhs[0] + pp.P)) is None
    assert dec(w[:3] + _limbs(lhs[1] + pp.P) + w[6:]) is None
    assert dec(w[:6] + _limbs(rhs[0] + pp.P) + w[9:]) is None
    # off the curve, and the identity
    assert dec(_words((1, 3), rhs)) is None
    assert dec(_words(lhs, (rhs[0], rhs[1] + 1))) is None
    assert dec(_words((0, 0), rhs)) is None and dec(_words(lhs, (0, 0))) is None
    # (1, 2) is on the curve: only the point rule decides
    assert dec(_words(G1, rhs)) == plonk.KzgAccumulator(G1, rhs)
    with pytest.raises(ValueError):
        dec(w[:11])


# ---- the committed fixtures: the contract's own stored words ---------------------------------------------------------
def _runs():
    with open(os.path.join(GOLDEN, "verifier_contract_runs.json")) as f:
        return json.load(f)


def _combined_verdict(kats, got):
    """the contract's decision from evm_pairing_points' pair: e(A, [1]_2) e(B, -[s]_2) = 1"""
    g2, s = contract_g2(kats)
    _, a, b = got
    return pp.pairing_check([pyref.aff_tuple(a), pyref.aff_tuple(b)], [g2, pp.g2_neg(s)])


@pytest.mark.parametrize("path", fixtures(), ids=lambda p: p.split("_")[-2])
def test_fixture_accumulator_is_valid_and_its_pairing_points_are_the_contracts(orc, kats, path):
    vk, instances, proof, _ = load_fixture(path)
    vp = contract_vp(kats)
    acc = plonk.accumulator_from_limbs(instances[0][:12])
    assert acc.lhs == pyref.ec_mul(acc.rhs, _tau(orc))
    assert plonk.verify_proof(BE, vp, vk, instances, proof, accumulator_indices=IDX) is None
    got = plonk.evm_pairing_points(BE, vp, vk, instances, proof, IDX)
    r, a, b = got
    stored = {int(v, 16) for v in _runs()[os.path.basename(path)]["stored_words"]}
    for v in (r,) + acc.lhs + acc.rhs + a + b:
        assert v in stored, hex(v)
    assert _combined_verdict(kats, got)
    # the fixture tool's limbs, which made these instances, are accumulator_to_limbs'
    assert make_k23_fixture.accumulator_limbs(_tau(orc), make_k23_fixture.ACCUMULATOR_SCALAR) == instances[0][:12]


def test_accumulator_indices_outside_the_instances_are_a_caller_error(kats):
    vk, instances, proof, _ = load_fixture(fixtures()[0])
    vp = contract_vp(kats)
    n = len(instances[0])
    for bad in ([(1, i) for i in range(12)], [(0, i) for i in range(n - 11, n + 1)], IDX[:11], [(0, -1)] + IDX[1:]):
        with pytest.raises(ValueError):
            plonk.verify_proof(BE, vp, vk, instances, proof, accumulator_indices=bad)
        with pytest.raises(ValueError):
            plonk.verify_proofs(BE, vp, [(vk, instances, proof, bad)])


# ---- the contract's verdicts on proofs with other accumulators --------------------------------------------------------
def _accumulator_runs():
    with open(os.path.join(GOLDEN, "accumulator_contract_runs.json")) as f:
        rec = json.load(f)
    vk, _, _, _ = load_fixture(os.path.join(GOLDEN, rec["fixture"]))
    return [(name, vk, [[int(v, 16) for v in run["instances"]]], bytes.fromhex(run["proof"]), run) for name, run in sorted(rec["runs"].items())]


def test_accumulator_check_gives_the_contracts_verdicts(kats):
    vp = contract_vp(kats)
    want = {"other_valid_accumulator": None, "lhs_tau_plus_one": "accumulator", "lhs_off_curve": "accumulator_encoding"}
    runs = _accumulator_runs()
    assert sorted(name for name, *_ in runs) == sorted(want)
    for name, vk, instances, proof, run in runs:
        got = plonk.verify_proof(BE, vp, vk, instances, proof, accumulator_indices=IDX)
        assert (None if got is None else got.kind) == want[name], (name, got)
        assert (got is None) == run["accepted"], name
        assert plonk.verify_proof(BE, vp, vk, instances, proof) is None, name        # halo2's check alone accepts all three
        pts = plonk.evm_pairing_points(BE, vp, vk, instances, proof, IDX)
        if isinstance(pts, plonk.ProofFailure):
            assert pts == got, name
            continue
        assert _combined_verdict(kats, pts) == (got is None), name
        if run["accepted"]:
            stored = {int(v, 16) for v in run["stored_words"]}
            acc = plonk.accumulator_from_limbs(instances[0][:12])
            assert all(v in stored for v in (pts[0],) + pts[1] + pts[2] + acc.lhs + acc.rhs), name
    # one batch with the fixture as a step-like item without indices: the one-at-a-time verdicts
    items = [(vk, inst, proof, IDX) for _, vk, inst, proof, _ in runs]
    fx_vk, fx_inst, fx_proof, _ = load_fixture(fixtures()[0])
    items.append((fx_vk, fx_inst, fx_proof))
    assert plonk.verify_proofs(BE, vp, items) == [plonk.verify_proof(BE, vp, *it[:3], accumulator_indices=it[3] if len(it) > 3 else None) for it in items]


# ---- two layers on the oracle engine ----------------------------------------------------------------------------------
def _seed0_vp(orc):
    return halo2.ParamsVerifierKZG(orc.g1_generator(), pp.g2_limbs(pp.G2_GEN), orc.srs_s_g2().reshape(16))


def _inner(orc):
    """a halo2lib-shaped snark over the Poseidon transcript at k = 8: (vk, instances, proof)"""
    k, inst = 8, [5, 6, 7]
    cs = circuits.halo2lib_shape(4, 2)
    fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, lookup_bits=4, groups=30, num_gate_advice=4, num_lookup_advice=2)
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    return plonk.verifying_key(pk), [inst], plonk.create_proof(E, pk, [inst], adv, SeededRng(5), poseidon.PoseidonTranscriptWrite(pk.vk_digest))


def _outer(acc, inner_instances):
    """an aggregation-shaped proof over the EVM transcript at k = 7 whose instances are acc's 12 limbs, then the inner instances"""
    k = 7
    inst = plonk.accumulator_to_limbs(acc) + inner_instances[0]
    cs = circuits.aggregation_shape()
    fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, lookup_bits=3, groups=20)
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    return plonk.verifying_key(pk), [inst], plonk.create_proof(E, pk, [inst], [adv], SeededRng(6), EvmTranscriptWrite(pk.vk_digest))


def test_two_layers_carry_the_inner_snarks_accumulator(orc):
    vp = _seed0_vp(orc)
    vk, instances, proof = _inner(orc)
    acc = plonk.succinct_verify(BE, vp, vk, instances, proof, transcript_read=poseidon.PoseidonTranscriptRead)
    assert isinstance(acc, plonk.KzgAccumulator)
    assert acc.lhs == pyref.ec_mul(acc.rhs, _tau(orc))                # (s W', W')
    assert plonk.aggregate_accumulators(BE, [acc]) == acc
    assert plonk.aggregate_accumulators(BE, [acc], transcript=poseidon.PoseidonTranscriptWrite(9)) == acc
    big = bytearray(proof); big[-96:-64] = pp.R.to_bytes(32, "little")   # the last evaluation = r
    assert plonk.succinct_verify(BE, vp, vk, instances, bytes(big), transcript_read=poseidon.PoseidonTranscriptRead).kind == "transcript"
    ovk, oinst, oproof = _outer(acc, instances)
    assert plonk.verify_proof(BE, vp, ovk, oinst, oproof, accumulator_indices=IDX) is None
    # one bit of the inner proof's last evaluation: the proof still reads, its accumulator no longer holds
    bad = bytearray(proof); bad[-96] ^= 1
    bad_acc = plonk.succinct_verify(BE, vp, vk, instances, bytes(bad), transcript_read=poseidon.PoseidonTranscriptRead)
    assert isinstance(bad_acc, plonk.KzgAccumulator) and bad_acc.lhs != pyref.ec_mul(bad_acc.rhs, _tau(orc))
    ovk, oinst, oproof = _outer(bad_acc, instances)
    assert plonk.verify_proof(BE, vp, ovk, oinst, oproof) is None
    assert plonk.verify_proof(BE, vp, ovk, oinst, oproof, accumulator_indices=IDX).kind == "accumulator"


# ---- several accumulators ---------------------------------------------------------------------------------------------
def _passes(orc, acc):
    return BE.pairing_check_batch([pp.g1_limbs(acc.lhs), pp.g1_limbs(acc.rhs)],
                                  [pp.g2_limbs(pp.G2_GEN), pp.g2_limbs(pp.g2_neg(pp.g2_from_limbs(orc.srs_s_g2())))], 2)[0]


def test_aggregating_several_accumulators(orc):
    tau = _tau(orc)
    rng = random.Random(3)
    good = [_acc(rng, tau) for _ in range(3)]
    folded = plonk.aggregate_accumulators(BE, good)
    assert folded == plonk.aggregate_accumulators(BE, good, transcript=poseidon.PoseidonTranscriptWrite(0))
    assert folded not in good and _passes(orc, folded)
    other = plonk.aggregate_accumulators(BE, good, transcript=poseidon.PoseidonTranscriptWrite(1))
    assert other != folded and _passes(orc, other)
    # r^0 = 1: sum_i r^i acc_i with the r the default transcript squeezes
    T = poseidon.PoseidonTranscriptWrite(0)
    for a in good:
        T.common_ec_point(a.lhs); T.common_ec_point(a.rhs)
    r = T.squeeze_challenge()
    assert folded.rhs == pyref.msm([pow(r, i, pp.R) for i in range(3)], [a.rhs for a in good])
    for pos in range(3):
        accs = list(good)
        accs[pos] = _acc(rng, tau, good=False)
        assert not _passes(orc, accs[pos])
        assert not _passes(orc, plonk.aggregate_accumulators(BE, accs)), pos
    with pytest.raises(ValueError):
        plonk.aggregate_accumulators(BE, [])
