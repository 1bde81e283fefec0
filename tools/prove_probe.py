#!/usr/bin/env python3
"""Development probe (GPU box): create_proof of one circuit shape a few times with per-stage wall clock.
usage: prove_probe.py [aggregation|halo2lib] [k] [reps]"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spectre_b200 import circuits, halo2, plonk  # noqa: E402
from spectre_b200.transcript import EvmTranscriptWrite  # noqa: E402


def main():
    shape = sys.argv[1] if len(sys.argv) > 1 else "aggregation"
    k = int(sys.argv[2]) if len(sys.argv) > 2 else 23
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    be = halo2.Backend([0])
    srs = halo2.ParamsKZG.setup(be, k, plonk.fr_mont(0x5eed7a75)).precompute()
    inst = list(range(1, 15))
    if shape == "aggregation":
        cs = circuits.aggregation_shape()
        fixed, adv, copies = circuits.aggregation_witness(cs, k, inst, min(19, k - 2), 2000, seed=1, dense=True)
        adv = [adv]
    else:
        cs = circuits.halo2lib_shape()
        fixed, adv, copies = circuits.halo2lib_witness(cs, k, inst, min(16, k - 2), 500, seed=1)
    E = plonk.DeviceEngine(be, srs, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    g = np.random.default_rng(7)

    class Draw:
        def __call__(self, count):
            a = g.integers(0, 1 << 63, size=(count, 4), dtype=np.uint64); a[:, 3] &= np.uint64((1 << 60) - 1)
            return a

        def device_rows(self, E, count):
            return E.random_rows(count)
    draw = Draw() if os.environ.get("SPB_HOST_RNG", "0") == "0" else Draw().__call__
    for rep in range(reps):
        stages = {}
        t0 = time.perf_counter()
        plonk.create_proof(E, pk, [inst], adv, draw, EvmTranscriptWrite(pk.vk_digest), stages)
        E.sync()
        print(json.dumps({"rep": rep, "create_proof_s": round(time.perf_counter() - t0, 4), "stages": {a: round(b, 4) for a, b in stages.items()}}), flush=True)
    be.close()


if __name__ == "__main__":
    main()
