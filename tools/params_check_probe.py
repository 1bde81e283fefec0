#!/usr/bin/env python3
"""Cost of plonk.check_params on the first GPU: seed-0 params made on the device at each k, checked against the verifier
contract's G2 constants.

    python tools/params_check_probe.py [--ks 20 23 24] [--reps 5] [--out FILE]

Prints one JSON object (and writes it to --out when given): the GPU's name and power limit, queried in the same run, then per k
the wall seconds of check_params (median, min and max over --reps calls after one warm-up call, with the median of each stage
points / powers / lagrange) for:
  * clean: ParamsKZG.setup over the seed-0 secret, the trailer from the contract's constants; asserted to report [];
  * clean_tables: the same handle after precompute() (which builds no tables where they would take more than a quarter of the
    device: "tables_built" says whether it did, from the device memory precompute took);
  * bad_g / bad_g_lagrange: the same params re-uploaded with g[n/2] doubled, or with g_lagrange[n/2] + G; asserted to report
    [powers n/2, lagrange 0] and [lagrange n/2]: the bisections' cost.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as orc  # noqa: E402
from spectre_b200 import halo2, plonk  # noqa: E402
from tests import pypairing as pp  # noqa: E402
from tests import pyref  # noqa: E402
from tests.verify_common import contract_vp  # noqa: E402


def gpu_identity():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, watts = [s.strip() for s in out.split(",")]
        return name, float(watts)
    except Exception:
        return "unknown", None


def timed(be, params, vp, reps, want):
    E = plonk.DeviceEngine(be, params, params.k, 2)
    got = plonk.check_params(E, be, vp, seed=b"\x00" * 32)                 # warm-up, and the verdict
    assert [(f.kind, f.index) for f in got] == want, got
    walls, stages = [], []
    for i in range(reps):
        t = {}
        t0 = time.perf_counter()
        plonk.check_params(E, be, vp, seed=bytes([i + 1]) * 32, timings=t)
        walls.append(time.perf_counter() - t0)
        stages.append(t)
    return {"median_s": statistics.median(walls), "min_s": min(walls), "max_s": max(walls), "n": reps,
            "stages_median_s": {s: statistics.median(t[s] for t in stages) for s in stages[0]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[20, 23, 24])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "verifier_kats.json")) as f:
        kats = json.load(f)
    vp = contract_vp(kats)
    name, watts = gpu_identity()
    import torch
    orc.build()
    be = halo2.Backend([0])
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "ks": {}}
    for k in a.ks:
        n = 1 << k
        row = {}
        params = halo2.ParamsKZG.setup(be, k, orc.srs_tau())
        params.set_g2(vp.g2, vp.s_g2)
        row["clean"] = timed(be, params, vp, a.reps, [])
        g, gl = params.get_g(), params.get_g(basis=halo2.BASIS_G_LAGRANGE)
        free0 = torch.cuda.mem_get_info(0)[0]
        params.precompute()
        row["tables_built"] = torch.cuda.mem_get_info(0)[0] < free0 - (1 << 30)
        row["clean_tables"] = timed(be, params, vp, a.reps, [])
        del params
        mid = pp.fq_ints(g[n // 2])
        p = (mid[0], mid[1])
        bad = g.copy(); bad[n // 2] = pp.g1_limbs(pyref.ec_add(p, p))
        params = halo2.ParamsKZG.from_parts(be, k, bad, gl)
        params.set_g2(vp.g2, vp.s_g2)
        del bad
        row["bad_g"] = timed(be, params, vp, a.reps, [("powers", n // 2), ("lagrange", 0)])
        del params
        mid = pp.fq_ints(gl[n // 2])
        bad = gl.copy(); bad[n // 2] = pp.g1_limbs(pyref.ec_add((mid[0], mid[1]), pp.G1_GEN))
        params = halo2.ParamsKZG.from_parts(be, k, g, bad)
        params.set_g2(vp.g2, vp.s_g2)
        del bad, g, gl
        row["bad_g_lagrange"] = timed(be, params, vp, a.reps, [("lagrange", n // 2)])
        del params
        be.release_workspace()
        res["ks"][str(k)] = row
        print(json.dumps({str(k): row}), file=sys.stderr, flush=True)
    be.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
