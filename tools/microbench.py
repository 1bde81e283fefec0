#!/usr/bin/env python3
"""Device micro-benchmarks (run on the GPU box): modular-multiply throughput and NTT / MSM device times.
Prints one JSON object per line; used to fill DESIGN.md's INT32-pipe roofline and to steer optimisation."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spectre_b200 import halo2  # noqa: E402

R_MOD = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001


def rand_fr(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2**63, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 60) - 1)  # < 2^252 < r : valid residues
    return a


def main():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    be = halo2.Backend([0])
    what = sys.argv[1:] or ["modmul", "ntt"]
    if "modmul" in what:
        for field in ("fq", "fr"):
            for ilp in (1, 2, 4):
                for tpsm in (512, 1024, 2048):
                    be.bench_modmul(field, sms * tpsm, 200, ilp)
                    ms, rate = be.bench_modmul(field, sms * tpsm, 2000, ilp)
                    print(json.dumps({"bench": "modmul", "field": field, "ilp": ilp, "threads_per_sm": tpsm, "ms": round(ms, 3), "gmul_per_s": round(rate / 1e9, 2)}), flush=True)
    if "modmul_quick" in what:
        for field in ("fq",):
            for ilp, nm in ((2, "mul"), (0x102, "sqr")):
                for tpsm in (384, 512, 1024):
                    be.bench_modmul(field, sms * tpsm, 200, ilp)
                    ms, rate = be.bench_modmul(field, sms * tpsm, 2000, ilp)
                    print(json.dumps({"bench": "modmul", "op": nm, "field": field, "threads_per_sm": tpsm, "ms": round(ms, 3), "gop_per_s": round(rate / 1e9, 2),
                                      "lib": os.path.basename(halo2.LIB_PATH)}), flush=True)
    if "ntt" in what:
        import torch
        root = pow(7, (R_MOD - 1) >> 28, R_MOD)
        sizes = [int(a.split("=")[1]) for a in what if a.startswith("k=")] or [12, 16, 18, 20, 21, 22, 23, 24, 25, 26]
        for k in sizes:
            w = pow(root, 1 << (28 - k), R_MOD) * (1 << 256) % R_MOD
            omega = np.array([[(w >> (64 * j)) & (2**64 - 1) for j in range(4)]], dtype=np.uint64)
            t = torch.from_numpy(rand_fr(1 << k, k).view(np.int64)).cuda()
            times = []
            for it in range(6):
                be.best_fft_dev(t.data_ptr(), omega, k)
                times.append(be.last_device_ms)
            best = min(times[1:])
            n = 1 << k
            print(json.dumps({"bench": "ntt", "k": k, "ms": round(best, 4), "gelem_per_s": round(n / best / 1e6, 3),
                              "algo_GBps": round(n * 64 / best / 1e6, 1), "first_ms": round(times[0], 3)}), flush=True)
            del t
    be.close()


if __name__ == "__main__":
    main()
