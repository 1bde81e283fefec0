#!/usr/bin/env python3
"""Cost of a powers-of-tau update (ParamsKZG.contribute, spb_srs_contribute) on the first GPU, and a three-update chain check.

    python tools/params_update_probe.py [--ks 20 23 24] [--out FILE]

Prints one JSON object (and writes it to --out when given): the GPU's name and power limit, queried in the same run
(nvidia-smi --query-gpu=name,power.limit --format=csv), then per k, for seed-0 params made with ParamsKZG.setup and given the
seed-0 G2 trailer (the verifier contract's constants):
  * ops: the operation counts from the code, n scalar multiples for the scaling and (n/2) log2 n + n for g_to_lagrange;
  * wall_s: one contribute call, wall clock (the call ends in a device synchronise), and device_ms: the library's own device
    time of that call (first scaling launch to the end of g_to_lagrange, spb_last_device_ms);
  * scale_ms / g_to_lagrange_ms: device time of srs_scale_kernel and of the g_to_lagrange kernels (ec_lift, fr_powers,
    ec_ntt_stage, ec_ntt_finish), from torch.profiler in a second, profiled contribute call;
  * min_free_gib: the lowest free device memory seen during the timed call (polled every 5 ms);
  * chain_s: three plonk.contribute_params in a row, and check_s: plonk.check_params_updates on them, asserted to report [].
A contribute call at k = 10 first loads the kernels.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as orc  # noqa: E402
from spectre_b200 import halo2, plonk  # noqa: E402
from tests.verify_common import contract_vp  # noqa: E402

G2L = ("ec_lift_kernel", "fr_powers_kernel", "ec_ntt_stage_kernel", "ec_ntt_finish_kernel")


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True, timeout=30).stdout
    return out.strip().splitlines()[1] if len(out.strip().splitlines()) > 1 else out.strip()


class MinFree:
    """the lowest torch.cuda.mem_get_info(0) free bytes while the block runs"""

    def __enter__(self):
        import torch
        self.torch, self.low, self.stop = torch, torch.cuda.mem_get_info(0)[0], threading.Event()

        def poll():
            while not self.stop.is_set():
                self.low = min(self.low, self.torch.cuda.mem_get_info(0)[0])
                time.sleep(0.005)
        self.thread = threading.Thread(target=poll)
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()
        self.low = min(self.low, self.torch.cuda.mem_get_info(0)[0])


def kernel_ms(params, t):
    """device ms of the scaling and of g_to_lagrange in one profiled contribute call"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        new = params.contribute(t)
    del new
    scale = g2l = 0.0
    seen = set()
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        dt = e.time_range.elapsed_us()
        if "srs_scale_kernel" in e.name:
            scale += dt
            seen.add("srs_scale_kernel")
        for name in G2L:
            if name in e.name:
                g2l += dt
                seen.add(name)
    assert "srs_scale_kernel" in seen and "ec_ntt_stage_kernel" in seen, "the profiler saw none of the library's kernels: %s" % sorted(seen)
    return scale / 1000.0, g2l / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[20, 23, 24])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "verifier_kats.json")) as f:
        vp = contract_vp(json.load(f))
    res = {"gpu": gpu_identity(), "ks": {}}
    orc.build()
    be = halo2.Backend([0])
    t = plonk.fr_mont(0x1234567890abcdef)
    warm = halo2.ParamsKZG.setup(be, 10, orc.srs_tau())
    warm.set_g2(vp.g2, vp.s_g2)
    warm.contribute(t)
    del warm
    for k in a.ks:
        n = 1 << k
        row = {"ops": {"scale_multiples": n, "g_to_lagrange_multiples": (n // 2) * k + n}}
        params = halo2.ParamsKZG.setup(be, k, orc.srs_tau())
        params.set_g2(vp.g2, vp.s_g2)
        with MinFree() as mem:
            t0 = time.perf_counter()
            new = params.contribute(t)
            row["wall_s"] = time.perf_counter() - t0
        row["device_ms"] = be.last_device_ms
        row["min_free_gib"] = mem.low / 2 ** 30
        del new
        row["scale_ms"], row["g_to_lagrange_ms"] = kernel_ms(params, t)
        t0 = time.perf_counter()
        p, updates = params, []
        for _ in range(3):
            p, u = plonk.contribute_params(be, p)
            updates.append(u)
        row["chain_s"] = time.perf_counter() - t0
        del params
        t0 = time.perf_counter()
        got = plonk.check_params_updates(plonk.DeviceEngine(be, p, k, 2), be, vp, updates)
        row["check_s"] = time.perf_counter() - t0
        assert got == [], got
        del p
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
