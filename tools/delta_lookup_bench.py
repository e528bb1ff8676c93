"""Updatable-index costs on the GPU (DeltaRMIIndex, DESIGN §19): lookups over base + delta, inserts, compaction.

Base: the §11 headline index, linear,linear 2^20 over 200M uniform uint64 keys below 2^63 (tools/lookup_bench.py's
seeded generator).  Inserted keys: uniform over the same range, device-resident batches.
  lookups     for delta sizes 0, 2^16, 2^20 and 2^23: lower_bound, upper_bound and equal_range of DeltaRMIIndex, of the
              base index alone, and torch.searchsorted (left, right, both) over the merged array, on 2^27 random
              queries drawn from the logical key set.  Every delta answer is checked against torch.searchsorted.  The
              delta-count kernel's own time (k_delta_count) comes from a torch.profiler pass after the timed calls.
  inserts     one insert of 2^16 and of 2^20 keys into deltas of 2^20 and 2^23 keys (host clock around the synchronous
              call; a fresh delta of the given size for every timed insert).
  compaction  200M + 2^20 keys: merged_keys() (merge + the sortedness check), the check alone (a data set of the same
              size wrapped in place), retrain, evaluate, and RMIIndex creation over the merged keys.
Per call: the median of --iters timed calls after --warmup untimed ones (CUDA events around each).  Prints one JSON
line, with the card's name and power limit read in the same run.

    python tools/delta_lookup_bench.py [--keys 200000000] [--queries 134217728] [--iters 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import rmi_b200  # noqa: E402
from lookup_bench import gen_keys, gpu_info, time_call  # noqa: E402

SPEC, BF = "linear,linear", 1 << 20
DELTAS = [0, 1 << 16, 1 << 20, 1 << 23]


def device_batch(g, m):
    b = torch.sort(torch.randint(0, (1 << 63) - 1, (m,), dtype=torch.int64, device="cuda", generator=g))[0]
    torch.cuda.synchronize()
    return rmi_b200.RMITrainingData.from_device(b.data_ptr(), m, rmi_b200.KEY_U64, 0, keep_alive=b), b


def count_kernel_ms(fn) -> float:
    """mean milliseconds of k_delta_count per call of fn, from a profiled run of 5 calls"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "k_delta_count" in e.name]
    return round(sum(ts) / 1000.0 / 5, 4) if ts else float("nan")


def lookups(keys, base, nq, iters, warmup):
    g = torch.Generator(device="cuda")
    g.manual_seed(99)
    n = keys.numel()
    first = torch.empty(nq, dtype=torch.int64, device="cuda")
    last = torch.empty_like(first)
    s = torch.cuda.current_stream().cuda_stream
    out = {}
    for m in DELTAS:
        d = rmi_b200.DeltaRMIIndex(base)
        ins = []
        if m:
            ds, b = device_batch(g, m)
            d.insert(ds)
            ins.append(b)
            del ds
        allk = torch.sort(torch.cat([keys, *ins]))[0] if m else keys
        q = allk[torch.randint(0, n + m, (nq,), device="cuda", generator=g)]
        p = q.data_ptr()
        calls = {
            "delta_lower_bound": lambda: d.lower_bound_device(p, nq, first.data_ptr(), 0, s),
            "delta_upper_bound": lambda: d.upper_bound_device(p, nq, last.data_ptr(), 0, s),
            "delta_equal_range": lambda: d.equal_range_device(p, nq, first.data_ptr(), last.data_ptr(), 0, s),
            "base_lower_bound": lambda: base.lower_bound_device(p, nq, first.data_ptr(), 0, s),
            "base_upper_bound": lambda: base.upper_bound_device(p, nq, last.data_ptr(), 0, s),
            "base_equal_range": lambda: base.equal_range_device(p, nq, first.data_ptr(), last.data_ptr(), 0, s),
            "searchsorted_left": lambda: torch.searchsorted(allk, q),
            "searchsorted_right": lambda: torch.searchsorted(allk, q, right=True),
            "searchsorted_left_right": lambda: (torch.searchsorted(allk, q), torch.searchsorted(allk, q, right=True)),
        }
        e = {k: round(time_call(fn, iters, warmup), 4) for k, fn in calls.items()}
        want_lo, want_hi = torch.searchsorted(allk, q), torch.searchsorted(allk, q, right=True)
        d.lower_bound_device(p, nq, first.data_ptr(), 0, s)
        exact = bool(torch.equal(first, want_lo))
        d.upper_bound_device(p, nq, last.data_ptr(), 0, s)
        exact &= bool(torch.equal(last, want_hi))
        first.fill_(-1)
        last.fill_(-1)
        d.equal_range_device(p, nq, first.data_ptr(), last.data_ptr(), 0, s)
        exact &= bool(torch.equal(first, want_lo)) and bool(torch.equal(last, want_hi))
        assert exact, f"delta {m}: an answer differs from torch.searchsorted"
        e["exact"] = exact
        if m:
            e["count_kernel_lower_ms"] = count_kernel_ms(calls["delta_lower_bound"])
            e["count_kernel_equal_range_ms"] = count_kernel_ms(calls["delta_equal_range"])
        e["probes_per_query_model"] = math.ceil(math.log2(m + 1))
        e["count_bytes_per_query_model"] = {"one_bound": 16, "equal_range": 24} if m else 0
        out[str(m)] = e
        d.close()
        del allk, q, want_lo, want_hi, ins
        torch.cuda.empty_cache()
    return out


def inserts(base, iters):
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    out = {}
    for m in (1 << 20, 1 << 23):
        for b in (1 << 16, 1 << 20):
            ts = []
            for _ in range(iters):
                d = rmi_b200.DeltaRMIIndex(base)
                ds, keep = device_batch(g, m)
                d.insert(ds)
                bs, bkeep = device_batch(g, b)
                t0 = time.perf_counter()
                d.insert(bs)
                ts.append((time.perf_counter() - t0) * 1e3)
                d.close()
                del ds, keep, bs, bkeep
            out[f"delta_{m}_batch_{b}_ms"] = round(float(np.median(ts)), 4)
            out[f"delta_{m}_batch_{b}_merge_bytes_model"] = 2 * (m + b) * 8
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, round((time.perf_counter() - t0) * 1e3, 3)


def compaction(keys, base, trained, reps):
    g = torch.Generator(device="cuda")
    g.manual_seed(77)
    n, m = keys.numel(), 1 << 20
    d = rmi_b200.DeltaRMIIndex(base)
    ds, keep = device_batch(g, m)
    d.insert(ds)
    phases = {"merge_and_check": [], "check_alone": [], "retrain": [], "evaluate": [], "index_create": []}
    for _ in range(reps):
        merged, t = timed(d.merged_keys)
        phases["merge_and_check"].append(t)
        big = torch.cat([keys, keys[:m]])   # n + m keys, wrapped in place: rmi_dataset_wrap_device's check alone
        torch.cuda.synchronize()
        w, t = timed(lambda: rmi_b200.RMITrainingData.from_device(big.data_ptr(), n + m, rmi_b200.KEY_U64, 0))
        phases["check_alone"].append(t)
        w.close()
        del big
        r, t = timed(lambda: rmi_b200.train(merged, SPEC, BF, counts=False))
        phases["retrain"].append(t)
        e, t = timed(lambda: rmi_b200.evaluate(trained, merged, counts=False))
        phases["evaluate"].append(t)
        idx, t = timed(lambda: rmi_b200.RMIIndex(r, merged))
        phases["index_create"].append(t)
        idx.close()
        merged.close()
    d.close()
    res = {k: round(float(np.median(v)), 3) for k, v in phases.items()}
    res["merge_bytes_model"] = 2 * (n + m) * 8
    res["keys"] = n + m
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("delta_lookup_bench needs a CUDA device")
    res = {"tool": "delta_lookup_bench", **gpu_info(), "spec": SPEC, "branching_factor": BF, "keys": a.keys,
           "queries": a.queries}
    keys = gen_keys("u64", a.keys)
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), a.keys, rmi_b200.KEY_U64, 0, keep_alive=keys)
    trained = rmi_b200.train(ds, SPEC, BF, counts=False)
    base = rmi_b200.RMIIndex(trained, ds)
    res["lookups"] = lookups(keys, base, a.queries, a.iters, a.warmup)
    res["inserts"] = inserts(base, max(3, a.iters // 4))
    res["compaction"] = compaction(keys, base, trained, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
