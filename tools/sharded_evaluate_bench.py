"""rmi_evaluate over range-partitioned keys: evaluate_sharded's one-call form (rmi_shard_evaluate) against rmi_evaluate
of the whole key set on one GPU, in the same run.

Workload: the section 13.4 headline, the tables of linear,linear 2^20 trained on 200M uniform uint64 keys below 2^63
(bench.py's seeded generator), evaluated on the same keys split evenly over the ranks.  Per call: median of --iters
calls after --warmup untimed ones; the per-phase split is the result's phase_device_ns (CUDA events: upload,
boundaries with their all-reduce, error pass with its all-reduce, statistics).  Asserts that the sharded result equals
rmi_evaluate's in every field.  Prints one JSON line (rank 0).

    python tools/sharded_evaluate_bench.py                      # world 1: one-rank NCCL communicator
    torchrun --nproc-per-node G tools/sharded_evaluate_bench.py  # NCCL, one GPU per rank
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

PHASES = ("upload", "boundaries", "error_pass", "statistics")
FIELDS = ("model_avg_error", "model_avg_l2_error", "model_avg_log2_error", "model_max_log2_error", "model_max_error",
          "model_max_error_idx", "num_rmi_rows", "num_data_rows")


def same(a, b) -> bool:
    bits = lambda v: np.asarray(v, dtype=np.float64).view(np.uint64)   # noqa: E731
    return (np.array_equal(a.last_layer_max_l1s, b.last_layer_max_l1s) and np.array_equal(a.l1_counts, b.l1_counts)
            and np.array_equal(bits(a.l1_params), bits(b.l1_params))
            and all(np.array_equal(bits(getattr(a, f)), bits(getattr(b, f))) for f in FIELDS))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("sharded_evaluate_bench needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl")
    n = a.keys
    g = torch.Generator(device=dev)
    g.manual_seed(42)
    keys = torch.sort(torch.randint(0, (1 << 63) - 1, (n,), dtype=torch.int64, device=dev, generator=g))[0]
    full = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, dev.index, keep_alive=keys)
    trained = rmi_b200.train(full, "linear,linear", 1 << 20, counts=False)
    lo, hi = sharded.slab_bounds(n, rank, world)
    data = sharded.ShardedTrainingData(keys[lo:hi].clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
    if sharded.native_comm(None, dev, single_rank_ok=True) is None:
        raise SystemExit("the one-call form needs NCCL (libnccl.so.2)")

    first = {}

    def run(name, fn):
        """(phase_device_ns, device_time_ns) of every timed call; each result is compared and dropped, so that its
        page-locked buffers are recycled as in a serving loop."""
        for _ in range(a.warmup):
            fn()
        wall, res, equal = [], [], True
        for _ in range(a.iters):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            r = fn()
            wall.append((time.perf_counter() - t0) * 1e3)
            res.append((list(r.phase_device_ns), r.device_time_ns))
            first.setdefault(name, r)
            equal = equal and same(r, first[name])
        return res, float(np.median(wall)), equal

    shard_res, shard_wall, eq1 = run("sharded", lambda: sharded.evaluate_sharded(trained, data, native=True))
    single_res, single_wall, eq2 = run("single", lambda: rmi_b200.evaluate(trained, full))
    med = lambda rs, q: float(np.median([r[0][q] for r in rs])) / 1e6   # noqa: E731
    res = {
        "world": world, "keys": n, "spec": "linear,linear", "branching_factor": 1 << 20, "iters": a.iters,
        "warmup": a.warmup, "version": rmi_b200.version(),
        "sharded_phase_ms": {p: round(med(shard_res, q), 4) for q, p in enumerate(PHASES)},
        "sharded_device_ms": round(float(np.median([r[1] for r in shard_res])) / 1e6, 4),
        "sharded_wall_ms": round(shard_wall, 4),
        "rmi_evaluate_phase_ms": {p: round(med(single_res, q), 4) for q, p in enumerate(PHASES)},
        "rmi_evaluate_device_ms": round(float(np.median([r[1] for r in single_res])) / 1e6, 4),
        "rmi_evaluate_wall_ms": round(single_wall, 4),
        "allreduce_bytes": 8 * (1 << 20) * (1 if data._ends_all[:, 4].all() else 2),
        "equal": eq1 and eq2 and same(first["sharded"], first["single"]),
    }
    if world > 1:
        t = torch.tensor([int(res["equal"])], dtype=torch.int64, device=dev)
        dist.all_reduce(t)
        res["equal"] = int(t.item()) == world
    if rank == 0:
        print(json.dumps({**gpu_info(), **res}))
    if world > 1:
        dist.destroy_process_group()
    if not res["equal"]:
        raise SystemExit("the sharded evaluation differs from rmi_evaluate")
    return res


if __name__ == "__main__":
    main()
