"""spectre_b200.plonk.verify_proof / verify_proofs on the GPU: the device's multiexp and pairing decide the committed fixtures
with the verifier contracts' G2 constants, and accept what create_proof makes on the device, over the seed-0 SRS and over a
setup with another secret."""
import random

import pytest

from spectre_b200 import circuits, halo2, plonk, poseidon
from spectre_b200.transcript import EvmTranscriptRead, EvmTranscriptWrite
from tests import pypairing as pp
from tests.gpu_common import be  # noqa: F401
from tests.plonk_oracle_engine import SeededRng
from tests.verify_common import alterations, contract_vp, fixtures, load_fixture

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("path", fixtures(), ids=lambda p: p.split("_")[-2])
def test_fixture_accepted_and_the_contracts_rejections_rejected(be, kats, path):
    vk, instances, proof, own = load_fixture(path)
    assert plonk.verify_proof(be, contract_vp(kats), vk, instances, proof) is None
    for name, vp, vk2, inst2, proof2 in alterations(kats, vk, instances, proof, own):
        got = plonk.verify_proof(be, vp, vk2, inst2, proof2)
        assert got is not None and got.kind == "opening", name


def _shape(name):
    if name == "aggregation":
        k, inst = 7, [3, 1, 4]
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, lookup_bits=3, groups=20)
        return cs, k, inst, fixed, [adv], copies
    if name == "sync_step":
        k, inst = 8, [5, 6, 7]
        cs = circuits.halo2lib_shape(4, 2)
        fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, lookup_bits=4, groups=30, num_gate_advice=4, num_lookup_advice=2)
        return cs, k, inst, fixed, adv, copies
    k, inst = 7, [7, 9]
    cs = circuits.wide_shape(3)
    fixed, adv, copies = circuits.wide_witness(cs, k, inst, lookup_bits=3, groups=20)
    return cs, k, inst, fixed, adv, copies


def _params(be, k, secret):
    """ParamsKZG.setup over `secret` (an int), its G2 trailer set to ([1]_2, [secret]_2) computed by the reference"""
    params = halo2.ParamsKZG.setup(be, k, plonk.fr_mont(secret))
    with pytest.raises(ValueError, match="set_g2 first"):
        params.verifier_params()
    params.set_g2(pp.g2_limbs(pp.G2_GEN), pp.g2_limbs(pp.g2_mul(pp.G2_GEN, secret)))
    return params


@pytest.mark.parametrize("shape", ["aggregation", "sync_step", "wide"])
@pytest.mark.parametrize("transcript", ["evm", "poseidon"])
def test_device_proofs_are_accepted(be, orc, shape, transcript):
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    cs, k, inst, fixed, adv, copies = _shape(shape)
    params = _params(be, k, tau)
    assert pp.g2_from_limbs(params.get_g2()[1]) == pp.g2_from_limbs(orc.srs_s_g2())
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    W, Rd = (poseidon.PoseidonTranscriptWrite, poseidon.PoseidonTranscriptRead) if transcript == "poseidon" else (EvmTranscriptWrite, EvmTranscriptRead)
    proof = plonk.create_proof(E, pk, [inst], adv, SeededRng(3), W(pk.vk_digest))
    vp, vk = params.verifier_params(), plonk.verifying_key(pk)
    assert plonk.verify_proof(be, vp, vk, [inst], proof, transcript_read=Rd) is None
    bad = bytearray(proof); bad[len(bad) // 2] ^= 1
    assert plonk.verify_proof(be, vp, vk, [inst], bytes(bad), transcript_read=Rd) is not None


def test_proof_over_a_setup_with_another_secret(be, orc):
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    secret = random.Random(91).randrange(2, pp.R)
    assert secret != tau
    cs, k, inst, fixed, adv, copies = _shape("aggregation")
    params = _params(be, k, secret)
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    proof = plonk.create_proof(E, pk, [inst], adv, SeededRng(8), EvmTranscriptWrite(pk.vk_digest))
    vk = plonk.verifying_key(pk)
    assert plonk.verify_proof(be, params.verifier_params(), vk, [inst], proof) is None
    # the seed-0 trailer does not open this proof
    other = halo2.ParamsVerifierKZG(params.verifier_params().g, pp.g2_limbs(pp.G2_GEN), orc.srs_s_g2().reshape(16))
    assert plonk.verify_proof(be, other, vk, [inst], proof).kind == "opening"


class _CountingBackend:
    """the device backend, counting the kernel launches of its pairing_check_batch calls"""

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


def test_verify_proofs_on_a_batch_gives_each_proofs_verdict(be, orc):
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    cs, k, inst, fixed, adv, copies = _shape("aggregation")
    params = _params(be, k, tau)
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    vk, vp = plonk.verifying_key(pk), params.verifier_params()
    items = [(vk, [inst], plonk.create_proof(E, pk, [inst], adv, SeededRng(100 + i), EvmTranscriptWrite(pk.vk_digest))) for i in range(32)]
    flip = bytearray(items[3][2]); flip[11 * 64 + 5] ^= 1
    off = bytearray(items[9][2]); off[63] ^= 1
    items[3] = (vk, [inst], bytes(flip))                                  # an evaluation bit
    items[9] = (vk, [inst], bytes(off))                                   # a point off the curve
    items[14] = (vk, [[inst[0] + 1] + inst[1:]], items[14][2])            # another public input
    items[20] = (vk, [inst], items[20][2][:-1])                           # truncated
    items[27] = (vk, [inst], items[27][2] + b"\x00")                      # a trailing byte
    one_at_a_time = [plonk.verify_proof(be, vp, *it) for it in items]
    counting = _CountingBackend(be)
    batch = plonk.verify_proofs(counting, vp, items)
    assert batch == one_at_a_time
    assert [i for i, v in enumerate(batch) if v is not None] == [3, 9, 14, 20, 27]
    assert [batch[i].kind for i in (3, 9, 14, 20, 27)] == ["opening", "transcript", "opening", "transcript", "transcript"]
    single = _CountingBackend(be)
    assert plonk.verify_proofs(single, vp, items[:1]) == [None]
    assert counting.calls == single.calls == 1 and counting.pairing_launches == single.pairing_launches == 3
