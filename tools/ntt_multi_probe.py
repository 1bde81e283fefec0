#!/usr/bin/env python3
"""In-process multi-device NTT timing probe: wall clock and device time of spb_ntt over every visible GPU."""
import ctypes, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spectre_b200 import halo2
from bench import rand_fr, R_MOD
g = torch.cuda.device_count()
be = halo2.Backend(list(range(g)))
root = pow(7, (R_MOD - 1) >> 28, R_MOD)
for k in (22, 24):
    w = pow(root, 1 << (28 - k), R_MOD) * (1 << 256) % R_MOD
    omega = np.array([[(w >> (64 * j)) & (2**64 - 1) for j in range(4)]], dtype=np.uint64)
    host = torch.from_numpy(rand_fr(1 << k, k).view(np.int64)).pin_memory()
    arr = host.numpy().view(np.uint64)
    for it in range(3):
        t0 = time.perf_counter()
        rc = be.lib.spb_ntt(be.ctx, arr.ctypes.data_as(ctypes.c_void_p), k, omega.ctypes.data_as(ctypes.c_void_p))
        print("k", k, "iter", it, "wall ms", round((time.perf_counter() - t0) * 1e3, 3), "device ms", round(be.last_device_ms, 3), flush=True)
be.close()
