"""The configuration search over range-partitioned keys against the replica search, in one run, on one GPU.

    python tools/sharded_optimize_bench.py [--n 200000000] [--profile fast|memory|disk]

Prints one JSON line: the wall time of find_pareto_efficient_configs_sharded (world 1, one-call batches over a one-rank
NCCL communicator) and the sum of its per-group device time, the wall time of api.find_pareto_efficient_configs on one
replica of the same keys, both fronts compared entry by entry, and the card's name and power limit read in the same run.
Keys: n uniform uint64 keys drawn and sorted on the device (seeded)."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200_000_000)
    ap.add_argument("--profile", default=os.environ.get("RMI_OPTIMIZER_PROFILE", ""))
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    if a.profile:
        os.environ["RMI_OPTIMIZER_PROFILE"] = a.profile
    else:
        os.environ.pop("RMI_OPTIMIZER_PROFILE", None)
    import rmi_b200
    from rmi_b200 import sharded
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29517")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1)
    g = torch.Generator(device="cuda").manual_seed(a.seed)
    keys = torch.randint(-(1 << 63), (1 << 63) - 1, (a.n,), dtype=torch.int64, device="cuda", generator=g)
    keys = (keys.view(torch.int64) ^ (-(1 << 63))).sort().values ^ (-(1 << 63))   # sorted as unsigned
    data = sharded.ShardedTrainingData(keys, halo_capacity=0)
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), a.n, rmi_b200.KEY_U64, 0, keep_alive=keys)

    device_ns = [0]
    groups = [0]
    inner = sharded.train_stats_batch_sharded

    def timed(*args, **kw):
        res = inner(*args, **kw)
        device_ns[0] += sum(r.device_time_ns for r in res)
        groups[0] += 1
        return res
    sharded.train_stats_batch_sharded = timed
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    front_s = sharded.find_pareto_efficient_configs_sharded(data, 10, native=True)
    t_sharded = time.perf_counter() - t0
    t0 = time.perf_counter()
    front_r = rmi_b200.find_pareto_efficient_configs(ds, 10)
    t_replica = time.perf_counter() - t0

    def key(f):
        return (f["models"], f["branching_factor"], f["size"])
    same = [key(x) == key(y) and x["max_log2_error"] == y["max_log2_error"] and
            abs(x["average_log2_error"] - y["average_log2_error"]) <= 1e-10 * abs(y["average_log2_error"])
            for x, y in zip(front_s, front_r)]
    print(json.dumps({
        "n": a.n, "profile": a.profile or "default", "world": 1,
        "sharded_wall_s": round(t_sharded, 3), "sharded_device_s": round(device_ns[0] / 1e9, 3), "sharded_groups": groups[0],
        "replica_wall_s": round(t_replica, 3),
        "fronts_equal": len(front_s) == len(front_r) and all(same), "entries_equal": same,
        "front_sharded": [key(f) for f in front_s], "front_replica": [key(f) for f in front_r],
        "card": card()}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
