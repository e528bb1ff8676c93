"""Lookups over range-partitioned keys: ShardedRMIIndex.lower_bound (the one-call form, rmi_shard_index_lower_bound)
against RMIIndex.lower_bound over the whole key set on one GPU.

Workload: the section 11 headline index, linear,linear 2^20 over 200M uniform uint64 keys below 2^63 (bench.py's
seeded generator), split evenly over the ranks; every rank submits 2^27 random present keys drawn from the whole key
set.  Per call: median of --iters calls after --warmup untimed ones, CUDA events.  Reports the per-phase split
(route + pack, count exchange with its host read, query exchange, search, answer exchange, gather), the total,
aggregate G queries/s, the bytes exchanged, fallbacks, and the single-GPU RMIIndex in the same run.  Prints one JSON
line (rank 0).

    python tools/sharded_lookup_bench.py                      # world 1: one-rank NCCL communicator
    torchrun --nproc-per-node G tools/sharded_lookup_bench.py  # NCCL, one GPU per rank
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rmi_b200  # noqa: E402
from rmi_b200 import sharded  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the measurement itself does not depend on it
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def timed(fn, iters: int, warmup: int) -> list[float]:
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27, help="per rank")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("sharded_lookup_bench needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl")
    n, nq = a.keys, a.queries
    g = torch.Generator(device=dev)
    g.manual_seed(42)
    keys = torch.sort(torch.randint(0, (1 << 63) - 1, (n,), dtype=torch.int64, device=dev, generator=g))[0]
    full = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, dev.index, keep_alive=keys)
    trained = rmi_b200.train(full, "linear,linear", 1 << 20, counts=False)
    lo, hi = sharded.slab_bounds(n, rank, world)
    data = sharded.ShardedTrainingData(keys[lo:hi].clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
    idx = sharded.ShardedRMIIndex(trained, data)
    comm = sharded.native_comm(None, dev, single_rank_ok=True)
    if comm is None:
        raise SystemExit("the one-call form needs NCCL (libnccl.so.2)")
    g.manual_seed(1234 + rank)
    q = keys[torch.randint(0, n, (nq,), device=dev, generator=g)]
    out = torch.empty(nq, dtype=torch.int64, device=dev)
    fb = torch.zeros(1, dtype=torch.int64, device=dev)
    L = rmi_b200.load_library()
    stream = torch.cuda.current_stream(dev).cuda_stream

    def one_call():
        rmi_b200.api._check(L.rmi_shard_index_lower_bound(idx.index._h, comm, q.data_ptr(), nq, out.data_ptr(), None,
                                                          C.c_void_p(stream)))

    phases = {p: [] for p in sharded.LOOKUP_PHASES}
    for _ in range(a.warmup):
        one_call()
    totals = []
    for _ in range(a.iters):
        totals += timed(one_call, 1, 0)
        st = idx.index.last_stats()
        for p, ms in st["phase_ms"].items():
            phases[p].append(ms)
    fb.zero_()
    rmi_b200.api._check(L.rmi_shard_index_lower_bound(idx.index._h, comm, q.data_ptr(), nq, out.data_ptr(),
                                                      fb.data_ptr(), C.c_void_p(stream)))
    exact = bool(torch.equal(out, torch.searchsorted(keys, q)))
    st = idx.index.last_stats()
    # single GPU, whole key set, same queries
    plain = rmi_b200.RMIIndex(trained, full)
    plain_ms = float(np.median(timed(lambda: plain.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), 0, stream),
                                     a.iters, a.warmup)))
    total_ms = float(np.median(totals))
    kb = 8
    res = {
        "world": world, "keys": n, "queries_per_rank": nq, "spec": "linear,linear", "branching_factor": 1 << 20,
        "iters": a.iters, "warmup": a.warmup, "version": rmi_b200.version(),
        "phase_ms": {p: round(float(np.median(v)), 4) for p, v in phases.items()},
        "total_ms": round(total_ms, 4),
        "aggregate_gq_per_s": round(world * nq / total_ms / 1e6, 3),
        "bytes_sent_to_peers": (nq - st["queries_kept"]) * kb + (st["queries_searched"] - st["queries_kept"]) * 8,
        "bytes_moved_incl_self": nq * kb + st["queries_searched"] * 8,
        "fallbacks": int(fb.item()), "exact": exact,
        "rmi_index_lower_bound_ms": round(plain_ms, 4),
        "overhead_vs_rmi_index_ms": round(total_ms - plain_ms, 4),
    }
    if world > 1:
        t = torch.tensor([res["fallbacks"], int(exact)], dtype=torch.int64, device=dev)
        dist.all_reduce(t)
        res["fallbacks"], res["exact"] = int(t[0]), int(t[1]) == world
    if rank == 0:
        print(json.dumps({**gpu_info(), **res}))
    idx.close()
    plain.close()
    if world > 1:
        dist.destroy_process_group()
    return res


if __name__ == "__main__":
    main()
