#!/usr/bin/env python3
"""Cost of the KZG accumulator check on the first GPU: plonk.verify_proof on the committed K = 23 fixture with and without
accumulator_indices, and plonk.verify_proofs on batches of aggregation items.

    python tools/accumulator_probe.py [--reps 20] [--batch-reps 3] [--out FILE]

Prints one JSON object (and writes it to --out when given):
  * the GPU's name and power limit, queried in the same run;
  * verify_proof on tests/golden/aggregation_k23_proof.json with the verifier contract's G2 constants, without and with
    AGGREGATION_ACCUMULATOR_INDICES: wall ms per call, the multiexp's device ms and the pairing check's device ms (CUDA
    events, spb_last_device_ms), medians over --reps calls after one warm-up call;
  * verify_proofs on batches of 1, 64 and 1024 copies of that fixture, each with the accumulator indices: wall ms per batch,
    the summed multiexp device ms, the device ms of its one pairing call (two checks per item), and, for comparison, the
    device ms of a pairing call on the same items' opening checks alone; medians over --batch-reps batches.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spectre_b200 import halo2, plonk  # noqa: E402
from tests.verify_common import contract_vp, load_fixture  # noqa: E402
from tools.verify_probe import gpu_identity  # noqa: E402


class Timed:
    """the device backend with wall and device ms recorded per call, and the last pairing call's inputs kept"""

    def __init__(self, be):
        self.be, self.log, self.last_pairing = be, [], None

    def best_multiexp(self, coeffs, bases):
        t = time.perf_counter(); out = self.be.best_multiexp(coeffs, bases)
        self.log.append(("msm", (time.perf_counter() - t) * 1e3, self.be.last_device_ms))
        return out

    def pairing_check_batch(self, ps, qs, m):
        t = time.perf_counter(); out = self.be.pairing_check_batch(ps, qs, m)
        self.log.append(("pairing", (time.perf_counter() - t) * 1e3, self.be.last_device_ms))
        self.last_pairing = (ps, qs)
        return out


def timed_runs(tb, reps, call):
    rows = []
    for _ in range(reps):
        tb.log = []
        t = time.perf_counter()
        call()
        wall = (time.perf_counter() - t) * 1e3
        rows.append(dict(wall=wall, msm_dev=sum(r[2] for r in tb.log if r[0] == "msm"),
                         pairing_dev=sum(r[2] for r in tb.log if r[0] == "pairing")))
    return {key: statistics.median(r[key] for r in rows) for key in rows[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "verifier_kats.json")) as f:
        kats = json.load(f)
    name, watts = gpu_identity()
    be = halo2.Backend([0])
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "batch_reps": a.batch_reps}
    vk, instances, proof, _ = load_fixture(os.path.join(ROOT, "tests", "golden", "aggregation_k23_proof.json"))
    vp = contract_vp(kats)
    idx = plonk.AGGREGATION_ACCUMULATOR_INDICES
    tb = Timed(be)
    for key, ind in (("verify_proof_k23_ms", None), ("verify_proof_k23_with_accumulator_ms", idx)):
        call = lambda: plonk.verify_proof(tb, vp, vk, instances, proof, accumulator_indices=ind)
        assert call() is None                                                       # warm-up
        res[key] = timed_runs(tb, a.reps, lambda: call())
    res["verify_proofs_with_accumulator_ms"] = {}
    for n in (1, 64, 1024):
        items = [(vk, instances, proof, idx)] * n
        call = lambda: plonk.verify_proofs(tb, vp, items)
        assert call() == [None] * n                                                 # warm-up
        row = timed_runs(tb, a.batch_reps, call)
        ps, qs = (np.asarray(v, dtype=np.uint64).reshape(n, 2, 2, -1) for v in tb.last_pairing)   # item, check, pair
        opening_ps, opening_qs = ps[:, 0].reshape(2 * n, -1), qs[:, 0].reshape(2 * n, -1)
        dev = []
        for _ in range(a.batch_reps + 1):
            assert be.pairing_check_batch(opening_ps, opening_qs, 2) == [True] * n
            dev.append(be.last_device_ms)
        row["opening_checks_alone_pairing_dev"] = statistics.median(dev[1:])
        res["verify_proofs_with_accumulator_ms"][str(n)] = row
    be.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
