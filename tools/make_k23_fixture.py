#!/usr/bin/env python3
"""Produce tests/golden/aggregation_k23_proof.json (and, with --k 24, aggregation_k24_proof.json for the committee-update
verifier contract): a proof of the aggregation-shaped synthetic circuit at K = 23
(the size the reference's sync_step verifier contract is generated for), made by the proof driver bound to the CPU
ORACLE, then replayed through the reference's own verifier contract (tests/yul_harness.py) -- the fixture is only
written if the contract accepts it. Needs the reference's contracts/snark-verifiers and ~25 GiB of RAM (~10 minutes).

The GPU test tests/test_gpu_plonk.py::test_k23_proof_equals_the_contract_accepted_fixture regenerates the same proof
with the CUDA engine (same seed, same witness) and requires identical bytes.

usage: python tools/make_k23_fixture.py --contracts <reference checkout>/contracts/snark-verifiers [--k 23]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as orc  # noqa: E402
from spectre_b200 import plonk  # noqa: E402
from spectre_b200.transcript import EvmTranscriptWrite  # noqa: E402
from spectre_b200 import circuits as plonk_circuits
from tests import pyref, yul_harness  # noqa: E402
from tests.plonk_oracle_engine import OracleEngine, SeededRng  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
SEED, GROUPS = 23, 2000
ACCUMULATOR_SCALAR = 0xACC                  # rhs = ACCUMULATOR_SCALAR * G of the fixtures' accumulator
# K -> (contract, lookup bits of its range table, number of public inputs): config/sync_step_verifier_23.json,
# config/committee_update_verifier_24.json (SURVEY.md section 8 rows 4 and 5)
CONTRACTS = {23: ("sync_step_verifier", 19, "range_table_commit_k23_bits19"), 24: ("committee_update_verifier", 23, "range_table_commit_k24_bits23")}


def accumulator_limbs(tau, s):
    """12 instance words: (lhs.x, lhs.y, rhs.x, rhs.y) in three 88-bit limbs each, with lhs = tau * rhs -- a valid KZG
    accumulator for the seed-0 SRS, the form the aggregation circuit exposes (sync_step_verifier.sol:213-236)."""
    rhs = pyref.ec_mul((1, 2), s)
    return plonk.accumulator_to_limbs(plonk.KzgAccumulator(pyref.ec_mul(rhs, tau), rhs))


def inputs(k, kats):
    contract, bits, _ = CONTRACTS.get(k, ("sync_step_verifier", min(19, k - 2), None))
    sched = kats["transcript_schedule"][contract]
    tau = orc.fr_ints(orc.srs_tau().reshape(1, 4))[0]
    instances = accumulator_limbs(tau, ACCUMULATOR_SCALAR) + [0x5eed0001 + i for i in range(sched["num_instances"] - 12)]
    cs = plonk_circuits.aggregation_shape()
    fixed, adv, copies = plonk_circuits.aggregation_witness(cs, k, instances, bits, GROUPS, seed=SEED)
    return cs, tau, instances, fixed, adv, copies, int(sched["vk_digest"]), bits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=23)
    ap.add_argument("--contracts", required=True, help="the reference's contracts/snark-verifiers directory")
    args = ap.parse_args()
    with open(os.path.join(GOLDEN, "verifier_kats.json")) as f:
        kats = json.load(f)
    k = args.k
    t0 = time.time()
    cs, tau, instances, fixed, adv, copies, digest, bits = inputs(k, kats)
    print("witness %.1fs" % (time.time() - t0), flush=True)
    E = OracleEngine(k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=digest)
    print("keygen %.1fs" % (time.time() - t0), flush=True)
    T = EvmTranscriptWrite(pk.vk_digest)
    timings = {}
    proof = plonk.create_proof(E, pk, [instances], [adv], SeededRng(SEED), T, timings)
    print("proof %.1fs" % (time.time() - t0), {a: round(b, 1) for a, b in timings.items()}, flush=True)
    vk_points = pk.fixed_commitments + pk.sigma_commitments
    if k in CONTRACTS:
        contract, _, kat = CONTRACTS[k]
        want = tuple(int(v, 16) for v in kats[kat]["xy"])
        assert pk.fixed_commitments[1] == want, "range-table commitment differs from the contract's VK constant"
        ok, m = yul_harness.run_contract(args.contracts, contract, instances, proof, vk_points, tau, kats)
        print("contract accepted:", ok, m.precompile_counts, flush=True)
        assert ok and m.pairing_calls == 1, "the reference verifier contract rejected the proof"
        fixture = {"_source": "tools/make_k23_fixture.py --k %d: proof driver on the CPU oracle; accepted by contracts/snark-verifiers/%s.sol replayed by tests/yul_harness.py" % (k, contract),
                   "contract": contract, "k": k, "seed": SEED, "lookup_bits": bits, "groups": GROUPS, "instances": [hex(v) for v in instances], "vk_digest": str(digest),
                   "vk_points": [[hex(x), hex(y)] for x, y in vk_points], "proof": proof.hex()}
        out = os.path.join(GOLDEN, "aggregation_k%d_proof.json" % k)
        with open(out, "w") as f:
            json.dump(fixture, f, indent=1)
        print("wrote", os.path.normpath(out))


if __name__ == "__main__":
    main()
