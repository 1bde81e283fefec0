#!/usr/bin/env python3
"""Cost of proof verification on the first GPU: plonk.verify_proof on the committed K = 23 fixture, and the pairing check alone.

    python tools/verify_probe.py [--reps 20] [--out FILE]

Prints one JSON object (and writes it to --out when given):
  * the GPU's name and power limit, queried in the same run;
  * verify_proof on tests/golden/aggregation_k23_proof.json with the verifier contract's G2 constants: wall ms per call, split
    into the multiexp (wall and device ms), the pairing check (wall and device ms) and the rest (transcript replay and the
    quotient identity, host Python), median over --reps calls after one warm-up call;
  * spb_pairing_check_batch at m = 2 and n_checks in {1, 64, 1024, 8192} (balanced and unbalanced checks mixed): the device ms
    of the three kernels (CUDA events, spb_last_device_ms), median, min and max over --reps calls after two warm-up calls.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spectre_b200 import halo2, plonk  # noqa: E402
from tests import pypairing as pp  # noqa: E402
from tests import pyref  # noqa: E402
from tests.verify_common import contract_vp, load_fixture  # noqa: E402


def gpu_identity():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, watts = [s.strip() for s in out.split(",")]
        return name, float(watts)
    except Exception:
        return "unknown", None


class Timed:
    """the device backend with wall and device time recorded per call of the two entry points verify_proof uses"""

    def __init__(self, be):
        self.be, self.log = be, []

    def best_multiexp(self, coeffs, bases):
        t = time.perf_counter(); out = self.be.best_multiexp(coeffs, bases)
        self.log.append(("msm", (time.perf_counter() - t) * 1e3, self.be.last_device_ms))
        return out

    def pairing_check_batch(self, ps, qs, m):
        t = time.perf_counter(); out = self.be.pairing_check_batch(ps, qs, m)
        self.log.append(("pairing", (time.perf_counter() - t) * 1e3, self.be.last_device_ms))
        return out


def stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "verifier_kats.json")) as f:
        kats = json.load(f)
    name, watts = gpu_identity()
    import torch
    be = halo2.Backend([0])
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps}
    # device memory the driver takes for the kernels' per-thread stacks (local memory) on the first pairing call
    free0 = torch.cuda.mem_get_info(0)[0]
    be.pairing_check_batch(np.stack([pp.g1_limbs(pp.G1_GEN)] * 2), np.stack([pp.g2_limbs(pp.G2_GEN)] * 2), 2)
    res["first_call_device_memory_taken_mib"] = (free0 - torch.cuda.mem_get_info(0)[0]) / 2 ** 20

    vk, instances, proof, _ = load_fixture(os.path.join(ROOT, "tests", "golden", "aggregation_k23_proof.json"))
    vp = contract_vp(kats)
    tb = Timed(be)
    assert plonk.verify_proof(tb, vp, vk, instances, proof) is None            # warm-up
    rows = []
    for _ in range(a.reps):
        tb.log = []
        t = time.perf_counter()
        assert plonk.verify_proof(tb, vp, vk, instances, proof) is None
        wall = (time.perf_counter() - t) * 1e3
        msm = [r for r in tb.log if r[0] == "msm"]; pair = [r for r in tb.log if r[0] == "pairing"]
        rows.append(dict(wall=wall, msm_wall=sum(r[1] for r in msm), msm_dev=sum(r[2] for r in msm), pairing_wall=sum(r[1] for r in pair),
                         pairing_dev=sum(r[2] for r in pair)))
    res["verify_proof_k23_ms"] = {key: statistics.median(r[key] for r in rows) for key in rows[0]}
    res["verify_proof_k23_ms"]["transcript_and_host"] = statistics.median(r["wall"] - r["msm_wall"] - r["pairing_wall"] for r in rows)

    rng = random.Random(5)
    pool = []
    for i in range(8):
        s = rng.randrange(2, pp.R)
        p, q = pyref.ec_mul(pp.G1_GEN, rng.randrange(1, pp.R)), pp.g2_mul(pp.G2_GEN, rng.randrange(1, pp.R))
        q2 = pp.g2_mul(q, s) if i % 2 == 0 else pp.g2_mul(q, s + 1)
        pool.append((np.stack([pp.g1_limbs(pyref.ec_mul(p, s)), pp.g1_limbs((p[0], (-p[1]) % pp.P))]),
                     np.stack([pp.g2_limbs(q), pp.g2_limbs(q2)]), i % 2 == 0))
    res["pairing_check_batch_m2_device_ms"] = {}
    for n_checks in (1, 64, 1024, 8192):
        pick = [j % len(pool) for j in range(n_checks)]
        ps = np.concatenate([pool[i][0] for i in pick]); qs = np.concatenate([pool[i][1] for i in pick])
        want = [pool[i][2] for i in pick]
        for _ in range(2):
            assert be.pairing_check_batch(ps, qs, 2) == want
        dev = []
        for _ in range(a.reps):
            be.pairing_check_batch(ps, qs, 2)
            dev.append(be.last_device_ms)
        res["pairing_check_batch_m2_device_ms"][str(n_checks)] = stats(dev)
    be.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
