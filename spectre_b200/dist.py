"""Multi-rank glue for the sharded MSM (SURVEY.md 8e): one process per GPU, point-range sharding, no data-path
collective -- only the 96-byte partial sums are all-gathered and folded on the host (EC addition is not an NCCL
reduction op). Backend-agnostic (`nccl` on the GPU box, `gloo` in the CPU tests)."""
import numpy as np

from . import halo2
from .halo2 import MONT_RADIX, R_MOD


def shard_range(n, rank, world):
    """Contiguous point range [lo, hi) owned by `rank` (same split the in-process multi-device context uses)."""
    return n * rank // world, n * (rank + 1) // world


def fold_partials(partials, world, device=None, group=None):
    """partials: (count, 12) uint64 Jacobian partial sums of this rank -> (count, 12) folded over all ranks."""
    import torch
    import torch.distributed as dist
    partials = np.ascontiguousarray(partials, dtype=np.uint64).reshape(-1, 12)
    if world == 1:
        return partials
    t = torch.from_numpy(partials.view(np.int64).copy())
    if device is not None:
        t = t.to(device)
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t, group=group)
    allp = torch.stack(out).cpu().numpy().view(np.uint64)          # (world, count, 12)
    return halo2.g1_sum_batch(allp)                                 # one host call for the whole batch


_MONT = MONT_RADIX % R_MOD


def _mont_int(a):
    a = np.asarray(a, dtype=np.uint64).reshape(4)
    return int(a[0]) | int(a[1]) << 64 | int(a[2]) << 128 | int(a[3]) << 192


def _mont_limbs(m):
    return np.array([(m >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)


def sharded_grand_product(local_total, seeded_scan, rank, world, init=None, device=None, group=None):
    """Row-sharded running product (SURVEY.md 8e "grand product": one exchange of G partial products, then a local
    fix-up). Rank r owns a contiguous block of rows. local_total() -> (4,) Montgomery product of this rank's rows
    (spb_product_dev); seeded_scan(seed) runs z[i] = seed * prod_{j<i} a[j] over them (spb_grand_product_seeded_dev).
    Returns (this rank's seed, the product of all rows times `init`), both Montgomery limbs."""
    import torch
    import torch.distributed as dist
    total = np.ascontiguousarray(local_total(), dtype=np.uint64).reshape(4)
    if world > 1:
        t = torch.from_numpy(total.view(np.int64).copy())
        if device is not None:
            t = t.to(device)
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t, group=group)
        totals = [o.cpu().numpy().view(np.uint64) for o in out]
    else:
        totals = [total]
    rinv = pow(_MONT, -1, R_MOD)
    seed = _mont_int(init) if init is not None else _MONT            # Montgomery one
    seeds = []
    for tq in totals:                                                # mont(a) * mont(b) * R^-1 = mont(a b)
        seeds.append(seed)
        seed = seed * _mont_int(tq) % R_MOD * rinv % R_MOD
    seeded_scan(_mont_limbs(seeds[rank]))
    return _mont_limbs(seeds[rank]), _mont_limbs(seed)
