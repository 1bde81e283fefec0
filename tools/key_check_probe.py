#!/usr/bin/env python3
"""Development probe (GPU box): what the proving-key check costs on Spectre's keys, with the card it ran on.

    python tools/key_check_probe.py [--reps 2] [--no-k24] [--out FILE]

For the k = 20 sync-step key and the K = 23 aggregation key (bench.py's shapes and fixed columns, params with the default
window tables), on the first GPU:
  * plonk.check_pk on the resident key from keygen: wall time and its split (commitments / polys / cosets / sigma);
  * plonk.write_pk to a temporary directory, then read_pk of that file in turn unchecked (RawBytesUnchecked) and checked
    (RawBytes), `reps` times each, alternating; the file was just written, so it is read from the page cache;
  * check_pk on the key read back.
Then check_pk on the K = 24 aggregation key made per_part (no cosets), if it fits beside the probe's other buffers (--no-k24
skips it). Last, the sigma pass on keys where every usable cell is on a copy cycle (sigma_c[i] labels (c, i + 1 mod u)): every
entry takes the full decode, the cost spb_copy_mismatches_dev pays as well, at K = 23 with 3 columns and k = 20 with 21.
Prints one JSON document (and writes it to --out)."""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import make_case  # noqa: E402
from spectre_b200 import halo2, plonk  # noqa: E402
from tools.srs_read_probe import gpu_identity  # noqa: E402

SECRET = plonk.fr_mont(0x5eed7a75)


def timed(E, fn):
    E.sync(); t0 = time.perf_counter()
    out = fn()
    E.sync()
    return out, time.perf_counter() - t0


def check(E, pk):
    stages = {}
    failures, t = timed(E, lambda: plonk.check_pk(E, pk, timings=stages))
    return {"failures": len(failures), "check_pk_s": round(t, 4), "stages_s": {a: round(b, 4) for a, b in stages.items()}}


def per_key(torch, be, name, k, reps, tmp):
    cs, _, fixed, _, _, copies, _ = make_case(torch, name, k, pin=False)
    params = halo2.ParamsKZG.setup(be, k, SECRET).precompute()
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    pk = plonk.keygen(E, cs, k, fixed, copies)
    del fixed
    row = {"shape": name, "k": k, "extended_k": E.extended_k, "fixed": cs.num_fixed, "permutation_columns": len(cs.permutation)}
    check(E, pk)                                                 # warm-up: tables, workspaces
    row["resident"] = check(E, pk)
    path = os.path.join(tmp, "%s_%d.pkey" % (name, k))
    plonk.write_pk(E, pk, path)
    row["file_bytes"] = os.path.getsize(path)
    del pk
    torch.cuda.empty_cache()
    reads = {"RawBytesUnchecked": [], "RawBytes": []}
    for _ in range(reps):
        for fmt in reads:
            back, t = timed(E, lambda: plonk.read_pk(E, cs, path, format=fmt))
            reads[fmt].append(round(t, 4))
            del back
            torch.cuda.empty_cache()
    row["read_pk_s"] = reads
    back = plonk.read_pk(E, cs, path, format="RawBytes")
    row["read_back"] = check(E, back)
    del back
    os.remove(path)
    del E, params
    be.release_workspace()
    torch.cuda.empty_cache()
    return row


def k24_per_part(torch, be):
    try:
        cs, _, fixed, _, _, copies, _ = make_case(torch, "aggregation_shape", 24, pin=False)
        params = halo2.ParamsKZG.setup(be, 24, SECRET).precompute()
        E = plonk.DeviceEngine(be, params, 24, cs.degree())
        pk = plonk.keygen(E, cs, 24, fixed, copies, cosets="per_part")
        del fixed
        check(E, pk)
        out = {"k": 24, "cosets": "per_part", **check(E, pk)}
        del pk, E, params
    except Exception as e:                                       # out of device memory: say so
        out = {"k": 24, "cosets": "per_part", "error": repr(e)[:300]}
    be.release_workspace()
    torch.cuda.empty_cache()
    return out


def dense_sigma(torch, be, k, cols, reps):
    """sigma where every usable cell is on a copy cycle: (c, i) -> (c, i + 1 mod u); the blinding rows stay fixed points"""
    n = 1 << k
    E = plonk.DeviceEngine(be, None, k, 4)
    u = n - 7
    perm = plonk.ConstraintSystem(0, cols, 0, [], [], [("advice", c) for c in range(cols)])
    ident = plonk.build_sigma(E, perm, k, [])
    sigma = []
    with torch.cuda.stream(E.stream):
        for s in ident:
            d = s.clone()
            d[:u - 1] = s[1:u]
            d[u - 1] = s[0]
            sigma.append(d)
    del ident
    zeros = [E.alloc(n) for _ in range(cols)]
    E.sigma_check(sigma, u, 16); E.copy_mismatches(zeros, sigma, u, 16)
    out = {"k": k, "columns": cols, "sigma_check_s": [], "copy_mismatches_s": []}
    for _ in range(reps):
        rep, t = timed(E, lambda: E.sigma_check(sigma, u, 16))
        assert all(total == 0 for kinds in rep for total, _ in kinds)
        out["sigma_check_s"].append(round(t, 4))
        rep, t = timed(E, lambda: E.copy_mismatches(zeros, sigma, u, 16))
        assert all(total == 0 for total, _ in rep)
        out["copy_mismatches_s"].append(round(t, 4))
    del sigma, zeros, E
    be.release_workspace()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--no-k24", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    name, watts = gpu_identity()
    doc = {"gpu": name, "power_limit_w": watts, "keys": []}
    be = halo2.Backend([0])
    with tempfile.TemporaryDirectory() as tmp:
        for shape, k in (("sync_step_shape", 20), ("aggregation_shape", 23)):
            doc["keys"].append(per_key(torch, be, shape, k, args.reps, tmp))
            print(json.dumps(doc["keys"][-1]), flush=True)
    if not args.no_k24:
        doc["k24"] = k24_per_part(torch, be)
        print(json.dumps(doc["k24"]), flush=True)
    doc["dense_sigma"] = [dense_sigma(torch, be, 23, 3, args.reps), dense_sigma(torch, be, 20, 21, args.reps)]
    be.close()
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
