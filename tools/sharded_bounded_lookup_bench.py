"""`--bounded` lookups over range-partitioned keys: ShardedBoundedRMIIndex.lower_bound and .predict (the one-call
forms, rmi_shard_index_lower_bound and rmi_shard_index_predict_collective) against BoundedRMIIndex over the whole key
set on one GPU and ShardedRMIIndex.lower_bound, in the same run.

Workload: 200M uniform uint64 keys below 2^63 (bench.py's seeded generator), split evenly over the ranks; for each line
size (8 and 64) the cache-fix spline over all keys and a linear,linear 2^20 RMI over its knots; every rank submits 2^27
random present keys.  The plain sharded index is the section 11 headline index (linear,linear 2^20 over the keys).
Per call: median of --iters calls after --warmup untimed ones, CUDA events; the per-phase split (route, count exchange
with its host read, query exchange, search, answer exchange, gather) of both sharded calls.  Prints one JSON line
(rank 0) with the card's name and power limit.

    python tools/sharded_bounded_lookup_bench.py                      # world 1: one-rank NCCL communicator
    torchrun --nproc-per-node G tools/sharded_bounded_lookup_bench.py  # NCCL, one GPU per rank
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rmi_b200  # noqa: E402
from rmi_b200 import sharded  # noqa: E402
from tools.sharded_lookup_bench import gpu_info, timed  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27, help="per rank")
    ap.add_argument("--lines", type=str, default="8,64")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("sharded_bounded_lookup_bench needs a CUDA device")
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
    lo, hi = sharded.slab_bounds(n, rank, world)
    data = sharded.ShardedTrainingData(keys[lo:hi].clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
    comm = sharded.native_comm(None, dev, single_rank_ok=True)
    if comm is None:
        raise SystemExit("the one-call forms need NCCL (libnccl.so.2)")
    g.manual_seed(1234 + rank)
    q = keys[torch.randint(0, n, (nq,), device=dev, generator=g)]
    out = torch.empty(nq, dtype=torch.int64, device=dev)
    err = torch.empty(nq, dtype=torch.int64, device=dev)
    L = rmi_b200.load_library()
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    def phase_medians(call, idx):
        phases = {p: [] for p in sharded.LOOKUP_PHASES}
        for _ in range(a.warmup):
            call()
        totals = []
        for _ in range(a.iters):
            totals += timed(call, 1, 0)
            for p, ms in idx.index.last_stats()["phase_ms"].items():
                phases[p].append(ms)
        return {p: round(float(np.median(v)), 4) for p, v in phases.items()}, round(float(np.median(totals)), 4)

    res = {"world": world, "keys": n, "queries_per_rank": nq, "spec": "linear,linear", "branching_factor": 1 << 20,
           "iters": a.iters, "warmup": a.warmup, "version": rmi_b200.version(), "lines": {}}
    for line in (int(x) for x in a.lines.split(",")):
        trained, knots = rmi_b200.train_bounded(full, "linear,linear", 1 << 20, line)
        idx = sharded.ShardedBoundedRMIIndex(trained, knots, line, data)
        h = idx.index._h

        def lower_bound():
            rmi_b200.api._check(L.rmi_shard_index_lower_bound(h, comm, q.data_ptr(), nq, out.data_ptr(), None, stream))

        def predict():
            rmi_b200.api._check(L.rmi_shard_index_predict_collective(h, comm, q.data_ptr(), nq, out.data_ptr(),
                                                                     err.data_ptr(), stream))

        lb_phases, lb_ms = phase_medians(lower_bound, idx)
        pr_phases, pr_ms = phase_medians(predict, idx)
        got, fb = idx.lower_bound(q, return_fallbacks=True, native=True)
        exact = bool(torch.equal(got, torch.searchsorted(keys, q)))
        one = rmi_b200.BoundedRMIIndex(trained, knots, line, full)
        one_lb = float(np.median(timed(lambda: one.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), 0,
                                                                       stream.value), a.iters, a.warmup)))
        one_pr = float(np.median(timed(lambda: one.predict_device(q.data_ptr(), nq, out.data_ptr(), err.data_ptr(),
                                                                   stream.value), a.iters, a.warmup)))
        r = {"knots": int(knots.shape[0]), "knot_rmi_max_error": int(trained.model_max_error),
             "halo_knots_per_side": sharded.knot_halo_width(trained),
             "lower_bound_phase_ms": lb_phases, "lower_bound_ms": lb_ms,
             "predict_phase_ms": pr_phases, "predict_ms": pr_ms,
             "fallbacks": fb, "exact": exact,
             "bounded_rmi_index_lower_bound_ms": round(one_lb, 4), "bounded_rmi_index_predict_ms": round(one_pr, 4)}
        if world > 1:
            t = torch.tensor([r["fallbacks"], int(exact)], dtype=torch.int64, device=dev)
            dist.all_reduce(t)
            r["fallbacks"], r["exact"] = int(t[0]), int(t[1]) == world
        res["lines"][str(line)] = r
        idx.close()
        one.close()
    # the plain sharded index over the same slabs and queries
    plain = sharded.ShardedRMIIndex(rmi_b200.train(full, "linear,linear", 1 << 20, counts=False), data)
    ph = plain.index._h
    res["sharded_rmi_index_lower_bound_phase_ms"], res["sharded_rmi_index_lower_bound_ms"] = phase_medians(
        lambda: rmi_b200.api._check(L.rmi_shard_index_lower_bound(ph, comm, q.data_ptr(), nq, out.data_ptr(), None,
                                                                  stream)), plain)
    plain.close()
    if rank == 0:
        print(json.dumps({**gpu_info(), **res}))
    if world > 1:
        dist.destroy_process_group()
    return res


if __name__ == "__main__":
    main()
