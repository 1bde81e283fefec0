#!/usr/bin/env python3
"""What lean proving keys (cosets="on_demand") and per-part keys (cosets="per_part") buy a process that holds Spectre's four
proving keys on one device, as ProverState::new does (sync-step and committee-update at k = 20, their aggregations at K = 23
and K = 24).

    python tools/prover_state_probe.py [--keys sync_step_shape:20,aggregation_shape:23,aggregation_shape:24] [--reps 3] [--no-four-keys] [--out FILE]

Per key shape, for every residency mode, on the first GPU:
  * the device bytes the key holds after keygen, from torch.cuda.mem_get_info (which also sees the library's own cudaMallocs;
    the library's workspaces are released before both readings), next to plonk.key_device_bytes and to the change of
    torch.cuda.memory_allocated. mem_get_info counts the whole device, so on a device shared with other processes, and at
    small k where the allocator's 2 MiB segments dominate, it can differ from the other two;
  * create_proof wall time, best of `reps` warm runs after one warm-up run, and whether every mode gives the same proof bytes.
Then the four-key run: the three smaller keys loaded lean (on_demand) and the K = 24 key per_part (or on_demand with
--k24-cosets on_demand), params at k = 20, 23 and 24 with the default window tables, then one proof per
key in turn, each after the library's workspaces are released. It records the free device memory after each load and before
each proof, the lowest free memory seen at each create_proof stage lap (the `timings` hook), each stage's time, and whether
each proof, the K = 24 one last, completed. If the K = 24 proof does not fit, it is repeated with only its own key and params loaded, and the
shortfall is its working set there minus the memory the four-key state left free. The committee-update k = 20 key uses the
sync-step shape as a stand-in. Witnesses and RNG are bench.py's. Prints one JSON document (and writes it to --out).
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import BENCH_VK_DIGEST, Draw, make_case  # noqa: E402
from spectre_b200 import halo2, plonk  # noqa: E402
from spectre_b200.transcript import EvmTranscriptWrite  # noqa: E402
from tools.srs_read_probe import gpu_identity  # noqa: E402

SECRET = plonk.fr_mont(0x5eed7a75)
GIB = float(1 << 30)


def free_bytes(torch, dev):
    torch.cuda.synchronize(dev)
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(dev)[0]


class FreeAtLaps(dict):
    """create_proof's `timings` dict that also keeps the lowest free device memory seen at each stage lap"""

    def __init__(self, torch, dev):
        super().__init__()
        self.torch, self.dev, self.low = torch, dev, {}

    def __setitem__(self, name, value):
        free = self.torch.cuda.mem_get_info(self.dev)[0]
        self.low[name] = min(self.low.get(name, free), free)
        super().__setitem__(name, value)


def prove(E, pk, inst, adv, timings=None):
    t0 = time.perf_counter()
    proof = plonk.create_proof(E, pk, [inst], adv, Draw(None, 7), EvmTranscriptWrite(pk.vk_digest), timings)
    E.sync()
    return proof, time.perf_counter() - t0


def per_key(torch, be, name, k, reps):
    cs, inst, fixed, _, pinned, copies, _ = make_case(torch, name, k)
    params = halo2.ParamsKZG.setup(be, k, SECRET).precompute()
    E = plonk.DeviceEngine(be, params, k, cs.degree())
    row, proofs = {"shape": name, "k": k, "extended_k": E.extended_k}, {}
    for mode in plonk.COSETS_MODES:
        be.release_workspace()
        before, before_torch = free_bytes(torch, E.dev), torch.cuda.memory_allocated(E.dev)
        t0 = time.perf_counter()
        pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=BENCH_VK_DIGEST, cosets=mode)
        E.sync()
        t_keygen = time.perf_counter() - t0
        be.release_workspace()
        held = before - free_bytes(torch, E.dev)
        held_torch = torch.cuda.memory_allocated(E.dev) - before_torch
        runs = [prove(E, pk, inst, pinned)[1] for _ in range(reps + 1)]
        proofs[mode], _ = prove(E, pk, inst, pinned)
        row[mode] = {"held_bytes": held, "held_gib": round(held / GIB, 3), "held_bytes_torch_allocated": held_torch,
                     "formula_bytes": plonk.key_device_bytes(cs, k, E.extended_k, mode),
                     "keygen_s": round(t_keygen, 3), "create_proof_s": round(min(runs[1:]), 4), "warm_runs_s": [round(t, 4) for t in runs[1:]],
                     "first_run_s": round(runs[0], 4)}
        del pk
    row["proofs_equal"] = all(p == proofs["resident"] for p in proofs.values())
    row["lean_extra_s"] = round(row["on_demand"]["create_proof_s"] - row["resident"]["create_proof_s"], 4)
    row["per_part_extra_s"] = round(row["per_part"]["create_proof_s"] - row["resident"]["create_proof_s"], 4)
    row["held_saved_share"] = round(1 - row["on_demand"]["held_bytes"] / row["resident"]["held_bytes"], 3)
    del E, params
    free_bytes(torch, 0)
    return row


def four_keys(torch, be, k24_cosets):
    dev = torch.device("cuda", be.devices[0])
    out = {"k24_cosets": k24_cosets, "free_at_start_gib": round(free_bytes(torch, dev) / GIB, 3)}
    params = {k: halo2.ParamsKZG.setup(be, k, SECRET).precompute() for k in (20, 23, 24)}
    out["free_after_params_gib"] = round(free_bytes(torch, dev) / GIB, 3)
    keys = []
    for label, name, k in (("sync_step", "sync_step_shape", 20), ("committee_update_stand_in", "sync_step_shape", 20),
                           ("sync_step_aggregation", "aggregation_shape", 23), ("committee_update_aggregation", "aggregation_shape", 24)):
        cs, inst, fixed, _, pinned, copies, _ = make_case(torch, name, k)
        E = plonk.DeviceEngine(be, params[k], k, cs.degree())
        pk = plonk.keygen(E, cs, k, fixed, copies, vk_digest=BENCH_VK_DIGEST, cosets=k24_cosets if k == 24 else "on_demand")
        del fixed
        be.release_workspace()
        keys.append((label, E, pk, inst, pinned))
        out["free_after_key_%s_gib" % label] = round(free_bytes(torch, dev) / GIB, 3)
    out["proofs"] = {}
    for label, E, pk, inst, pinned in keys:
        out["proofs"][label] = proof_with_laps(torch, be, dev, E, pk, inst, pinned)
    out["k24_proved"] = out["proofs"]["committee_update_aggregation"]["completed"]
    if not out["k24_proved"]:
        # the K = 24 proof's own working set, with every other key and params freed: what the four-key state lacks
        E, pk, inst, pinned = keys[-1][1:]
        del keys, params
        alone = out["k24_with_only_its_key_and_params"] = proof_with_laps(torch, be, dev, E, pk, inst, pinned)
        if alone["completed"]:
            alone["working_set_gib"] = round(alone["free_before_gib"] - alone["lowest_free_gib"], 3)
            out["k24_shortfall_gib"] = round(alone["working_set_gib"] - out["proofs"]["committee_update_aggregation"]["free_before_gib"], 3)
    return out


def proof_with_laps(torch, be, dev, E, pk, inst, pinned):
    """one create_proof after the library's workspaces of earlier proofs are released, as a server switching between key sizes
    would; -> free memory before it, the lowest free memory at each stage lap, and whether it completed"""
    be.release_workspace()
    rec = {"k": pk.k, "free_before_gib": round(free_bytes(torch, dev) / GIB, 3)}
    laps = FreeAtLaps(torch, dev)
    try:
        proof, t = prove(E, pk, inst, pinned, laps)
        rec.update(completed=True, create_proof_s=round(t, 4), proof_bytes=len(proof))
    except Exception as e:                                     # out of device memory: record how far it got
        rec.update(completed=False, error=repr(e)[:300])
    rec["lowest_free_gib_at_lap"] = {name: round(v / GIB, 3) for name, v in laps.low.items()}
    rec["stage_s"] = {name: round(v, 4) for name, v in laps.items()}
    rec["lowest_free_gib"] = round(min(laps.low.values()) / GIB, 3) if laps.low else None
    free_bytes(torch, dev)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default="sync_step_shape:20,aggregation_shape:23,aggregation_shape:24")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-four-keys", action="store_true")
    ap.add_argument("--k24-cosets", default="per_part", choices=plonk.COSETS_MODES[1:], help="residency of the K = 24 key in the four-key run")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    be = halo2.Backend([0])
    name, watts = gpu_identity()
    result = {"what": "proving-key residency: resident vs on_demand (lean) vs per_part cosets", "gpu": name, "power_limit_w": watts,
              "device_total_gib": round(torch.cuda.mem_get_info(0)[1] / GIB, 3), "keys": []}
    for spec in filter(None, args.keys.split(",")):
        shape, k = spec.split(":")
        result["keys"].append(per_key(torch, be, shape, int(k), args.reps))
        print(json.dumps(result["keys"][-1]), file=sys.stderr, flush=True)
    if not args.no_four_keys:
        result["four_keys_lean"] = four_keys(torch, be, args.k24_cosets)
    be.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
