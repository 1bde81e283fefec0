"""CPU-only tests of spectre_b200.plonk.verify_proof / verify_proofs with a pure-Python stand-in for its two device calls
(tests/verify_common.PyBackend: pyref.msm and tests/pypairing).

The committed fixtures are accepted with G2 taken only from the verifier contracts' constants -- tau is never given -- and the
four alterations the reference's contract rejected are rejected at the pairing. Malformed bytes are transcript failures. On
proofs the oracle engine makes, the verdict is the one the independent verifier (tests/plonk_verifier.py, tau known) gives,
before and after a corruption, for the aggregation, sync-step and wide shapes and for a Poseidon-transcript proof."""
import pytest

from spectre_b200 import circuits, halo2, plonk, poseidon
from spectre_b200.transcript import EvmTranscriptRead, EvmTranscriptWrite
from tests import plonk_verifier
from tests import pypairing as pp
from tests.plonk_oracle_engine import OracleEngine, SeededRng
from tests.verify_common import PyBackend, alterations, contract_vp, fixtures, load_fixture

BE = PyBackend()


@pytest.mark.parametrize("path", fixtures(), ids=lambda p: p.split("_")[-2])
def test_fixture_accepted_and_the_contracts_rejections_rejected_at_the_pairing(kats, path):
    vk, instances, proof, own = load_fixture(path)
    assert plonk.verify_proof(BE, contract_vp(kats), vk, instances, proof) is None
    for name, vp, vk2, inst2, proof2 in alterations(kats, vk, instances, proof, own):
        got = plonk.verify_proof(BE, vp, vk2, inst2, proof2)
        assert got is not None and got.kind == "opening", name


def test_malformed_proofs_are_transcript_failures(kats):
    vk, instances, proof, _ = load_fixture(fixtures()[0])
    vp = contract_vp(kats)
    off_curve = bytearray(proof); off_curve[63] ^= 1                      # y of the first point
    big = bytearray(proof); big[640:672] = pp.R.to_bytes(32, "big")      # the first evaluation = r
    for bad in (proof[:-1], proof + b"\x00", bytes(off_curve), bytes(big), proof[:100]):
        got = plonk.verify_proof(BE, vp, vk, instances, bad)
        assert got is not None and got.kind == "transcript", got
    with pytest.raises(ValueError):
        plonk.verify_proof(BE, vp, vk, instances + [[1]], proof)


def _oracle_proof(orc, shape, transcript="evm"):
    if shape == "aggregation":
        k, inst = 6, [11, 22, 39]
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, lookup_bits=3, groups=40)
        adv = [adv]
    elif shape == "sync_step":
        k, inst = 8, [5, 6, 7]
        cs = circuits.halo2lib_shape(4, 2)
        fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, lookup_bits=4, groups=30, num_gate_advice=4, num_lookup_advice=2)
    else:
        k, inst = 7, [7, 9]
        cs = circuits.wide_shape(3)
        fixed, adv, copies = circuits.wide_witness(cs, k, inst, lookup_bits=3, groups=20)
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    T = poseidon.PoseidonTranscriptWrite(pk.vk_digest) if transcript == "poseidon" else EvmTranscriptWrite(pk.vk_digest)
    return pk, [inst], plonk.create_proof(E, pk, [inst], adv, SeededRng(7), T)


def _seed0_vp(orc):
    g = orc.g1_generator()
    return halo2.ParamsVerifierKZG(g, pp.g2_limbs(pp.G2_GEN), orc.srs_s_g2().reshape(16))


def _reference_accepts(pk, instances, proof, tau, transcript_read):
    try:
        return plonk_verifier.verify(pk.cs, pk.k, pk.vk_digest, pk.fixed_commitments, pk.sigma_commitments, instances, proof, tau,
                                     transcript_read=transcript_read)
    except (AssertionError, ValueError):
        return False


@pytest.mark.parametrize("shape,transcript", [("aggregation", "evm"), ("sync_step", "evm"), ("wide", "evm"), ("sync_step", "poseidon")])
def test_oracle_proofs_get_the_independent_verifiers_verdict(orc, shape, transcript):
    pk, instances, proof = _oracle_proof(orc, shape, transcript)
    reader = poseidon.PoseidonTranscriptRead if transcript == "poseidon" else EvmTranscriptRead
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    vp, vk = _seed0_vp(orc), plonk.verifying_key(pk)
    bad = bytearray(proof); bad[len(bad) // 2] ^= 1
    wrong_input = [[instances[0][0] + 1] + instances[0][1:]]
    for inst, pr in ((instances, proof), (instances, bytes(bad)), (wrong_input, proof)):
        want = _reference_accepts(pk, inst, pr, tau, reader)
        got = plonk.verify_proof(BE, vp, vk, inst, pr, transcript_read=reader)
        assert (got is None) == want, (shape, transcript, got)
    assert _reference_accepts(pk, instances, proof, tau, reader)


def test_verify_proofs_gives_one_verdict_per_item_with_mixed_keys(orc, kats):
    """items with different keys (a fixture and an oracle proof of another shape) in one call: each verdict is verify_proof's"""
    pk, instances, proof = _oracle_proof(orc, "wide")
    vp = _seed0_vp(orc)
    assert pp.g2_from_limbs(vp.s_g2) == pp.g2_from_limbs(contract_vp(kats).s_g2)     # the fixtures were made over the seed-0 SRS
    vk = plonk.verifying_key(pk)
    fx_vk, fx_instances, fx_proof, _ = load_fixture(fixtures()[0])
    bad = bytearray(proof); bad[-1] ^= 1
    items = [(vk, instances, proof), (fx_vk, fx_instances, fx_proof), (vk, instances, bytes(bad)), (vk, instances, proof[:-3])]
    got = plonk.verify_proofs(BE, vp, items)
    assert got == [plonk.verify_proof(BE, vp, *it) for it in items]
    assert got[0] is None and got[1] is None and got[2] is not None and got[3].kind == "transcript"
