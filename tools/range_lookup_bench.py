"""Upper bounds and equal ranges on the GPU: RMIIndex.lower_bound / upper_bound / equal_range against
torch.searchsorted left, right and left + right (DESIGN §18).

Workloads (keys generated and sorted on the device with tools/lookup_bench.py's seeded generator):
  uniform      linear,linear 2^20 over 200M uniform uint64 keys below 2^63 (the §11 headline index)
  dups         the same keys with 5% duplicates: 5% of the positions take their predecessor's key
  bounded_8    the `--bounded` line-8 index over the uniform keys (key 0 dropped: cache-fix panics on it)
Query sets (2^27 each): random present keys, the same keys sorted, uniform over [min, max].  Per call: median
milliseconds of --iters CUDA-event-timed calls after --warmup untimed ones.  Every answer is checked against
torch.searchsorted, and the fallback counts are reported.  Prints one JSON line, with the card's name and power limit
read in the same run.  --sharded times ShardedRMIIndex.upper_bound at world 1 (the one-call form over a one-rank
NCCL communicator) against RMIIndex.upper_bound on the same index and random present queries, as
tools/sharded_lookup_bench.py does for lower_bound.

    python tools/range_lookup_bench.py [--keys 200000000] [--queries 134217728] [--iters 20] [--warmup 3] [--sharded]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import rmi_b200  # noqa: E402
from lookup_bench import gen_keys, gpu_info, time_call  # noqa: E402

SPEC, BF, LINE = "linear,linear", 1 << 20, 8


def with_duplicates(keys: torch.Tensor, frac: float = 0.05) -> torch.Tensor:
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    i = torch.randint(1, keys.numel(), (int(keys.numel() * frac),), device="cuda", generator=g)
    k = keys.clone()
    k[i] = keys[i - 1]   # still sorted: keys[i-1] <= keys[i] <= keys[i+1]
    return k


def build(name: str, keys: torch.Tensor):
    n = keys.numel()
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=keys)
    if name != "bounded_8":
        return rmi_b200.RMIIndex(rmi_b200.train(ds, SPEC, BF, counts=False), ds)
    knots = rmi_b200.cache_fix(keys.cpu().numpy().view("uint64"), LINE)
    kds = rmi_b200.RMITrainingData(knots[:, 0].copy())
    r = rmi_b200.train(kds, SPEC, BF, counts=False)
    r.num_data_rows = n
    return rmi_b200.BoundedRMIIndex(r, knots, LINE, ds)


def run(name: str, keys: torch.Tensor, nq: int, iters: int, warmup: int) -> dict:
    idx = build(name, keys)
    n = keys.numel()
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    present = keys[torch.randint(0, n, (nq,), device="cuda", generator=g)]
    qsets = {"present_random": present, "present_sorted": torch.sort(present)[0],
             "uniform": torch.randint(int(keys[0]), int(keys[-1]) + 1, (nq,), dtype=keys.dtype, device="cuda",
                                      generator=g)}
    first = torch.empty(nq, dtype=torch.int64, device="cuda")
    last = torch.empty_like(first)
    fb = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    res = {"workload": name, "spec": SPEC, "branching_factor": BF, "keys": n, "queries": {}}
    if name == "bounded_8":
        res["line_size"] = LINE
    for qname, q in qsets.items():
        p = q.data_ptr()
        calls = {
            "lower_bound": lambda: idx.lower_bound_device(p, nq, first.data_ptr(), 0, s),
            "upper_bound": lambda: idx.upper_bound_device(p, nq, last.data_ptr(), 0, s),
            "equal_range": lambda: idx.equal_range_device(p, nq, first.data_ptr(), last.data_ptr(), 0, s),
            "searchsorted_left": lambda: torch.searchsorted(keys, q),
            "searchsorted_right": lambda: torch.searchsorted(keys, q, right=True),
            "searchsorted_left_right": lambda: (torch.searchsorted(keys, q), torch.searchsorted(keys, q, right=True)),
        }
        e = {mode: round(time_call(fn, iters, warmup), 4) for mode, fn in calls.items()}
        want_lo, want_hi = torch.searchsorted(keys, q), torch.searchsorted(keys, q, right=True)
        fbs, exact = {}, True
        for mode in ("lower_bound", "upper_bound", "equal_range"):
            fb.zero_()
            first.fill_(-1)
            last.fill_(-1)
            if mode == "lower_bound":
                idx.lower_bound_device(p, nq, first.data_ptr(), fb.data_ptr(), s)
                exact &= bool(torch.equal(first, want_lo))
            elif mode == "upper_bound":
                idx.upper_bound_device(p, nq, last.data_ptr(), fb.data_ptr(), s)
                exact &= bool(torch.equal(last, want_hi))
            else:
                idx.equal_range_device(p, nq, first.data_ptr(), last.data_ptr(), fb.data_ptr(), s)
                exact &= bool(torch.equal(first, want_lo)) and bool(torch.equal(last, want_hi))
            fbs[mode] = int(fb.item())
        assert exact, f"{name}/{qname}: an answer differs from torch.searchsorted"
        e["fallbacks"] = fbs
        e["exact"] = exact
        e["equal_range_over_lower_bound"] = round(e["equal_range"] / e["lower_bound"], 3)
        e["upper_bound_speedup_vs_searchsorted_right"] = round(e["searchsorted_right"] / e["upper_bound"], 3)
        e["equal_range_speedup_vs_searchsorted_left_right"] = round(e["searchsorted_left_right"] / e["equal_range"], 3)
        res["queries"][qname] = e
    idx.close()
    return res


def run_sharded(keys: torch.Tensor, nq: int, iters: int, warmup: int) -> dict:
    from rmi_b200 import sharded
    n = keys.numel()
    full = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=keys)
    trained = rmi_b200.train(full, SPEC, BF, counts=False)
    data = sharded.ShardedTrainingData(keys.clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
    idx = sharded.ShardedRMIIndex(trained, data)
    plain = rmi_b200.RMIIndex(trained, full)
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    q = keys[torch.randint(0, n, (nq,), device="cuda", generator=g)]
    out = torch.empty(nq, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    got = idx.upper_bound(q, native=True)
    exact = bool(torch.equal(got, torch.searchsorted(keys, q, right=True)))
    assert exact, "ShardedRMIIndex.upper_bound differs from torch.searchsorted"
    del got
    ms_sharded = time_call(lambda: idx.upper_bound(q, native=True), iters, warmup)
    st = idx.index.last_stats()
    ms_plain = time_call(lambda: plain.upper_bound_device(q.data_ptr(), nq, out.data_ptr(), 0, s), iters, warmup)
    idx.close()
    plain.close()
    return {"workload": "sharded_world_1", "spec": SPEC, "branching_factor": BF, "keys": n, "queries": nq,
            "sharded_upper_bound_ms": round(ms_sharded, 4),
            "phase_ms": {p: round(v, 4) for p, v in st["phase_ms"].items()},
            "rmi_index_upper_bound_ms": round(ms_plain, 4), "exact": exact}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="uniform,dups,bounded_8")
    ap.add_argument("--sharded", action="store_true", help="ShardedRMIIndex.upper_bound at world 1 instead")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("range_lookup_bench needs a CUDA device")
    rmi_b200.load_library()
    out = {**gpu_info(), "version": rmi_b200.version(), "iters": a.iters, "warmup": a.warmup, "results": []}
    uniform = gen_keys("u64", a.keys)
    if a.sharded:
        out["results"].append(run_sharded(uniform, a.queries, a.iters, a.warmup))
        print(json.dumps(out))
        return out
    for name in a.workloads.split(","):
        keys = {"uniform": uniform, "dups": None, "bounded_8": None}[name]
        if name == "dups":
            keys = with_duplicates(uniform)
        elif name == "bounded_8":
            keys = uniform[uniform > 0].contiguous()
        out["results"].append(run(name, keys, a.queries, a.iters, a.warmup))
        del keys
        torch.cuda.empty_cache()
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
