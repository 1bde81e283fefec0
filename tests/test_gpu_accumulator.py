"""The KZG accumulator check of aggregation proofs on the GPU: the device's multiexp and pairing give the CPU verdicts on the
committed fixtures and on the contract's records, an inner snark's accumulator is carried into an outer proof entirely
through DeviceEngine, and a mixed batch of aggregation and step proofs is decided by one pairing launch sequence."""
import json
import os
import random

import pytest

from spectre_b200 import circuits, halo2, plonk, poseidon
from spectre_b200.transcript import EvmTranscriptWrite
from tests import pypairing as pp
from tests.gpu_common import be  # noqa: F401
from tests.plonk_oracle_engine import SeededRng
from tests.verify_common import GOLDEN, PyBackend, contract_vp, fixtures, load_fixture

pytestmark = pytest.mark.gpu
IDX = plonk.AGGREGATION_ACCUMULATOR_INDICES


def _cases():
    """(name, vk, instances, proof, the CPU verdict's kind): the fixtures and the contract's accumulator records"""
    out = []
    for path in fixtures():
        vk, instances, proof, _ = load_fixture(path)
        out.append((os.path.basename(path), vk, instances, proof, None))
    with open(os.path.join(GOLDEN, "accumulator_contract_runs.json")) as f:
        rec = json.load(f)
    want = {"other_valid_accumulator": None, "lhs_tau_plus_one": "accumulator", "lhs_off_curve": "accumulator_encoding"}
    vk = load_fixture(os.path.join(GOLDEN, rec["fixture"]))[0]
    for name, run in sorted(rec["runs"].items()):
        out.append((name, vk, [[int(v, 16) for v in run["instances"]]], bytes.fromhex(run["proof"]), want[name]))
    return out


def test_device_verdicts_on_the_fixtures_and_the_contracts_records(be, kats):
    vp = contract_vp(kats)
    cases = _cases()
    for name, vk, instances, proof, want in cases:
        got = plonk.verify_proof(be, vp, vk, instances, proof, accumulator_indices=IDX)
        assert (None if got is None else got.kind) == want, (name, got)
        assert plonk.verify_proof(be, vp, vk, instances, proof) is None, name
    name, vk, instances, proof, _ = cases[0]
    assert plonk.evm_pairing_points(be, vp, vk, instances, proof, IDX) == plonk.evm_pairing_points(PyBackend(), vp, vk, instances, proof, IDX)
    items = [(vk, instances, proof, IDX) for _, vk, instances, proof, _ in cases]
    assert [None if v is None else v.kind for v in plonk.verify_proofs(be, vp, items)] == [c[4] for c in cases]


# ---- two layers through DeviceEngine ----------------------------------------------------------------------------------
def _params(be, k, secret):
    params = halo2.ParamsKZG.setup(be, k, plonk.fr_mont(secret))
    params.set_g2(pp.g2_limbs(pp.G2_GEN), pp.g2_limbs(pp.g2_mul(pp.G2_GEN, secret)))
    return params


class _Layers:
    """the inner (halo2lib shape, k = 8) and outer (aggregation shape, k = 7) keys on the device, over params of one secret"""

    def __init__(self, be, secret):
        self.be = be
        self.inner_cs, self.outer_cs = circuits.halo2lib_shape(4, 2), circuits.aggregation_shape()
        self.inner_inst = [5, 6, 7]
        fixed, self.inner_adv, copies = circuits.halo2lib_witness(self.inner_cs, 8, self.inner_inst, lookup_bits=4, groups=30,
                                                                  num_gate_advice=4, num_lookup_advice=2)
        self.inner_params = _params(be, 8, secret)
        self.inner_E = plonk.DeviceEngine(be, self.inner_params, 8, self.inner_cs.degree())
        self.inner_pk = plonk.keygen(self.inner_E, self.inner_cs, 8, fixed, copies)
        self.outer_params = _params(be, 7, secret)
        self.outer_E = plonk.DeviceEngine(be, self.outer_params, 7, self.outer_cs.degree())
        # the aggregation witness puts instances only into advice and copy cells: one key for every accumulator
        fixed, _, copies = self._outer_witness([0] * 15)
        self.outer_pk = plonk.keygen(self.outer_E, self.outer_cs, 7, fixed, copies)
        self.vp = self.outer_params.verifier_params()

    def _outer_witness(self, inst):
        return circuits.aggregation_witness(self.outer_cs, 7, inst, lookup_bits=3, groups=20)

    def inner(self, seed, transcript=poseidon.PoseidonTranscriptWrite):
        pk = self.inner_pk
        return plonk.create_proof(self.inner_E, pk, [self.inner_inst], self.inner_adv, SeededRng(seed), transcript(pk.vk_digest))

    def succinct(self, proof, be=None):
        return plonk.succinct_verify(be or self.be, self.inner_params.verifier_params(), plonk.verifying_key(self.inner_pk),
                                     [self.inner_inst], proof, transcript_read=poseidon.PoseidonTranscriptRead)

    def outer(self, acc, seed):
        """(vk, instances, proof) of an outer proof whose instances are acc's limbs and then the inner instances"""
        inst = plonk.accumulator_to_limbs(acc) + self.inner_inst
        _, adv, _ = self._outer_witness(inst)
        pk = self.outer_pk
        return plonk.verifying_key(pk), [inst], plonk.create_proof(self.outer_E, pk, [inst], [adv], SeededRng(seed), EvmTranscriptWrite(pk.vk_digest))


@pytest.fixture(scope="module")
def layers(be, orc):
    return _Layers(be, orc.fr_ints(orc.srs_tau().reshape(1, 4))[0])


def test_two_layers_on_the_device(be, layers):
    proof = layers.inner(1)
    acc = layers.succinct(proof)
    assert isinstance(acc, plonk.KzgAccumulator)
    assert acc == layers.succinct(proof, PyBackend())
    assert plonk.aggregate_accumulators(be, [acc]) == acc
    vk, inst, outer = layers.outer(acc, 2)
    assert plonk.verify_proof(be, layers.vp, vk, inst, outer, accumulator_indices=IDX) is None
    # one bit of the inner proof's last evaluation
    bad = bytearray(proof); bad[-96] ^= 1
    bad_acc = layers.succinct(bytes(bad))
    assert isinstance(bad_acc, plonk.KzgAccumulator) and bad_acc == layers.succinct(bytes(bad), PyBackend())
    vk, inst, outer = layers.outer(bad_acc, 3)
    assert plonk.verify_proof(be, layers.vp, vk, inst, outer) is None
    assert plonk.verify_proof(be, layers.vp, vk, inst, outer, accumulator_indices=IDX).kind == "accumulator"


def test_inner_snark_under_another_secret_is_rejected(be, orc, layers):
    secret = random.Random(92).randrange(2, pp.R)
    other = _Layers(be, secret)
    acc = other.succinct(other.inner(4))
    vk, inst, outer = layers.outer(acc, 5)
    assert plonk.verify_proof(be, layers.vp, vk, inst, outer) is None
    assert plonk.verify_proof(be, layers.vp, vk, inst, outer, accumulator_indices=IDX).kind == "accumulator"
    # against its own secret's [s]_2 that accumulator holds
    g2, s_g2 = other.outer_params.get_g2()
    assert be.pairing_check_batch([pp.g1_limbs(acc.lhs), pp.g1_limbs(acc.rhs)], [g2, pp.g2_limbs(pp.g2_neg(pp.g2_from_limbs(s_g2)))], 2) == [True]


class _CountingBackend:
    """the device backend, counting its pairing_check_batch calls and their kernel launches"""

    def __init__(self, be):
        self.be, self.pairing_launches, self.calls = be, 0, 0

    def best_multiexp(self, coeffs, bases):
        return self.be.best_multiexp(coeffs, bases)

    def pairing_check_batch(self, ps, qs, m):
        before = self.be.kernel_launches
        out = self.be.pairing_check_batch(ps, qs, m)
        self.pairing_launches += self.be.kernel_launches - before
        self.calls += 1
        return out


def test_mixed_batch_of_aggregation_and_step_proofs(be, layers):
    acc = layers.succinct(layers.inner(10))
    bad = bytearray(layers.inner(11)); bad[-96] ^= 1
    bad_acc = layers.succinct(bytes(bad))
    step_vk = plonk.verifying_key(layers.inner_pk)
    items = []
    for i in range(32):
        if i % 3 == 2:                                                    # a step proof, no accumulator
            items.append((step_vk, [layers.inner_inst], layers.inner(200 + i, EvmTranscriptWrite)))
        else:
            items.append(layers.outer(acc, 100 + i) + (IDX,))
    vk, inst, proof, _ = items[4]
    off = plonk.accumulator_to_limbs(plonk.KzgAccumulator((1, 3), acc.rhs))
    items[4] = (vk, [off + inst[0][12:]], proof, IDX)                    # limbs that are not a curve point
    items[7] = layers.outer(bad_acc, 300) + (IDX,)                       # the accumulator of an invalid inner snark
    flip = bytearray(items[9][2]); flip[11 * 64 + 5] ^= 1
    items[9] = items[9][:2] + (bytes(flip), IDX)                         # an evaluation bit
    items[13] = items[13][:2] + (items[13][2][:-1], IDX)                 # truncated
    step_flip = bytearray(items[17][2]); step_flip[-129] ^= 1
    items[17] = (step_vk, items[17][1], bytes(step_flip))                # a bit of a step proof's last evaluation
    one_at_a_time = [plonk.verify_proof(be, layers.vp, *it[:3], accumulator_indices=it[3] if len(it) > 3 else None) for it in items]
    counting = _CountingBackend(be)
    batch = plonk.verify_proofs(counting, layers.vp, items)
    assert batch == one_at_a_time
    assert {i: v.kind for i, v in enumerate(batch) if v is not None} == {4: "accumulator_encoding", 7: "accumulator", 9: "opening",
                                                                         13: "transcript", 17: "opening"}
    assert counting.calls == 1 and counting.pairing_launches == 3
    # without indices, the aggregation items with accumulator faults pass: the default is halo2's check alone
    plain = plonk.verify_proofs(be, layers.vp, [it[:3] for it in items])
    assert plain[7] is None and plain[9].kind == "opening" and plain[13].kind == "transcript"
