#!/usr/bin/env python3
"""Cost of the checked params-file read: ParamsKZG::read_custom with RawBytes (every point validated on the device) against
RawBytesUnchecked, on the first GPU.

    python tools/srs_read_probe.py DIR [--ks 20,23] [--reps 3] [--keep]

Writes kzg_bn254_{k}.srs files into DIR with spb_srs_setup + spb_srs_write_file (k = 20: 128 MiB, K = 23: 1 GiB), then reads
each one `reps` times checked and `reps` times unchecked, alternating, and prints one JSON line: wall ms per read, the check
kernels' device ms of every checked read (CUDA events, spb_last_device_ms), and the GPU's name and power limit queried in the
same run. The files are read right after they are written, so the reads come from the page cache: this measures the cached-file
case, not a cold read from disk. The files are deleted afterwards unless --keep.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spectre_b200 import halo2  # noqa: E402

R_MOD = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001


def gpu_identity():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, watts = [s.strip() for s in out.split(",")]
        return name, float(watts)
    except Exception:
        return "unknown", None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--ks", default="20,23")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--keep", action="store_true")
    args = ap.parse_args()
    os.makedirs(args.dir, exist_ok=True)
    be = halo2.Backend([0])
    tau = pow(5, 0x5eed, R_MOD) * (1 << 256) % R_MOD
    secret = np.array([[(tau >> (64 * j)) & (2**64 - 1) for j in range(4)]], dtype=np.uint64)
    result = {"what": "ParamsKZG read_custom, RawBytes (checked) vs RawBytesUnchecked", "file_cache": "page-cached (read right after write)"}
    for k in [int(s) for s in args.ks.split(",")]:
        path = os.path.join(args.dir, "kzg_bn254_%d.srs" % k)
        params = halo2.ParamsKZG.setup(be, k, secret)
        params.write(path)
        del params
        rec = {"bytes": os.path.getsize(path), "checked_ms": [], "unchecked_ms": [], "check_kernel_ms": []}
        halo2.ParamsKZG.read_custom(be, path, "RawBytes")             # warm-up: module load, staging buffers, check slot
        for _ in range(args.reps):
            for fmt in ("RawBytes", "RawBytesUnchecked"):
                t0 = time.perf_counter()
                params = halo2.ParamsKZG.read_custom(be, path, fmt)
                ms = (time.perf_counter() - t0) * 1e3
                if fmt == "RawBytes":
                    rec["checked_ms"].append(round(ms, 2))
                    rec["check_kernel_ms"].append(round(be.last_device_ms, 3))
                else:
                    rec["unchecked_ms"].append(round(ms, 2))
                del params
        rec["check_kernel_share_of_checked_read"] = round(sum(rec["check_kernel_ms"]) / sum(rec["checked_ms"]), 4)
        result["k%d" % k] = rec
        if not args.keep:
            os.remove(path)
    name, watts = gpu_identity()
    result["gpu"] = name
    result["power_limit_w"] = watts
    be.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
