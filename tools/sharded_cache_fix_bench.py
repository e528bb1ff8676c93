"""The cache-fix spline over range-partitioned keys (cache_fix_sharded, DESIGN.md section 16) against
rmi_cache_fix_device of the whole key set on one GPU, in the same run.

Workload: 200M uniform uint64 keys below 2^63 (bench.py's seeded generator), line size 8, split evenly over the ranks.
Per phase: median of --iters runs after --warmup untimed ones, host clock around calls that end in a device
synchronisation (every scan reads its exit on the host): first scan (speculation, every stitch, resolve), joining
rounds (table all-gathers and re-scans), emit, knot gather (to every rank).  rmi_cache_fix_device is timed the same way
(scan, emit and the copy of the knots to the host).  Asserts that the knots are equal.  Prints one JSON line (rank 0).

    python tools/sharded_cache_fix_bench.py                                           # world 1
    python -m torch.distributed.run --nproc-per-node G tools/sharded_cache_fix_bench.py
With fewer GPUs than ranks the ranks share cuda:0 over gloo ("separate_gpus": false): the phases then do not run side
by side on separate devices, so the times are not those of a multi-GPU run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rmi_b200  # noqa: E402
from rmi_b200 import sharded  # noqa: E402
from tools.sharded_lookup_bench import gpu_info  # noqa: E402

PHASES = ("first_scan_s", "join_s", "emit_s", "gather_s")


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--line", type=int, default=8)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("sharded_cache_fix_bench needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    separate = torch.cuda.device_count() >= world
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")) if separate else 0)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl" if separate else "gloo")
    n = a.keys
    g = torch.Generator(device=dev)
    g.manual_seed(42)
    keys = torch.sort(torch.randint(1, (1 << 63) - 1, (n,), dtype=torch.int64, device=dev, generator=g))[0]
    lo, hi = sharded.slab_bounds(n, rank, world)
    data = sharded.ShardedTrainingData(keys[lo:hi].clone(), key_type=rmi_b200.KEY_U64, halo_capacity=1 << 16)
    runs, knots = [], None
    for it in range(a.warmup + a.iters):
        t = {}
        if world > 1:
            dist.barrier()
        knots = sharded.cache_fix_sharded(data, a.line, timings=t)
        if it >= a.warmup:
            runs.append(t)
    res = {"world": world, "separate_gpus": separate, "backend": dist.get_backend() if world > 1 else None,
           "keys": n, "line": a.line, "iters": a.iters, "warmup": a.warmup, "knots": int(knots.shape[0]),
           "join_rounds": [r["join_rounds"] for r in runs],
           "phase_ms": {p[:-2]: round(float(np.median([r[p] for r in runs])) * 1e3, 3) for p in PHASES},
           "version": rmi_b200.version()}
    res["total_ms"] = round(sum(res["phase_ms"].values()), 3)
    if rank == 0:
        full = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, dev.index, keep_alive=keys)
        single, want = [], None
        for it in range(a.warmup + a.iters):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            want = rmi_b200.cache_fix(full, a.line)
            if it >= a.warmup:
                single.append(time.perf_counter() - t0)
        full.close()
        res["rmi_cache_fix_device_ms"] = round(float(np.median(single)) * 1e3, 3)
        res["knots_equal"] = bool(np.array_equal(knots, want))
        print(json.dumps({**gpu_info(), **res}))
    ok = torch.tensor([int(res.get("knots_equal", True))], dtype=torch.int64)
    if world > 1:
        ok = ok.to(dev) if separate else ok
        dist.broadcast(ok, 0)
        dist.destroy_process_group()
    if not int(ok.item()):
        raise SystemExit("the sharded knots differ from rmi_cache_fix_device's")
    return res


if __name__ == "__main__":
    main()
