#!/usr/bin/env python3
"""Development probe (GPU box): plonk.check_witness on a clean witness of one circuit shape, with the wall clock of its gate,
lookup and copy-constraint stages, next to create_proof on the same key and witness. Prints one JSON line per repetition
and the card it ran on. The proof's blinding rows are constants and its random polynomial comes from the device's ChaCha20
stream, so the proof time is the prover's, not the host's.
usage: witness_check_probe.py [aggregation|halo2lib] [k] [reps]"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spectre_b200 import circuits, halo2, plonk  # noqa: E402
from spectre_b200.transcript import EvmTranscriptWrite  # noqa: E402


def main():
    shape = sys.argv[1] if len(sys.argv) > 1 else "aggregation"
    k = int(sys.argv[2]) if len(sys.argv) > 2 else 23
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    be = halo2.Backend([0])
    srs = halo2.ParamsKZG.setup(be, k, plonk.fr_mont(0x5eed7a75)).precompute()
    inst = list(range(1, 15))
    if shape == "aggregation":                                   # the bench's proof workload
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, min(19, k - 2), 2000, seed=1, dense=True)
        adv = [adv]
    else:
        cs = circuits.halo2lib_shape()
        fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, min(16, k - 2), 500, seed=1)
    E = plonk.DeviceEngine(be, srs, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    stages = {}

    def timed(name, fn):
        def run(*a, **kw):
            E.sync(); t = time.perf_counter()
            out = fn(*a, **kw)
            E.sync(); stages[name] = stages.get(name, 0.0) + time.perf_counter() - t
            return out
        return run
    E.graph_evaluate = timed("graph_evaluate", E.graph_evaluate)
    E.nonzero_rows = timed("gates_compaction", E.nonzero_rows)
    E.lookup_missing_rows = timed("lookup_membership", E.lookup_missing_rows)
    E.copy_mismatches = timed("copy_sigma_decode", E.copy_mismatches)
    for rep in range(reps):
        stages.clear()
        E.sync(); t0 = time.perf_counter()
        failures = plonk.check_witness(E, pk, [inst], adv, theta=0x1234)
        E.sync(); t_check = time.perf_counter() - t0
        t0 = time.perf_counter()
        plonk.create_proof(E, pk, [inst], adv, plonk.DeviceBulkRng(lambda count: plonk.fr_mont_rows([7] * count), 5), EvmTranscriptWrite(pk.vk_digest))
        E.sync(); t_proof = time.perf_counter() - t0
        print(json.dumps({"rep": rep, "shape": shape, "k": k, "failures": len(failures), "check_witness_s": round(t_check, 4),
                          "stages_s": {a: round(b, 4) for a, b in stages.items()}, "create_proof_s": round(t_proof, 4)}), flush=True)
    be.close()


if __name__ == "__main__":
    main()
