"""Costs of removals from updatable indexes on the GPU (DeltaRMIIndex.remove, DESIGN §19.5): lookups over
base ⊎ inserted ⊖ removed, removes, and compaction.

Base: the §11 headline index, linear,linear 2^20 over 200M uniform uint64 keys below 2^63 (tools/lookup_bench.py's
seeded generator), as in tools/delta_lookup_bench.py.  Inserted keys: uniform over the same range; removed keys: half
base keys and half inserted keys (all base keys when nothing is inserted), at distinct positions; device batches.
  lookups     for (m inserted, t removed) in (0, 2^16), (0, 2^20), (2^20, 2^20), (2^23, 2^20): lower_bound,
              upper_bound and equal_range of the delta with removals, of the insert-only delta with the same m, of the
              base index alone, and torch.searchsorted (left, right, both) over the logical keys, on 2^27 random
              queries drawn from the logical key set.  Every answer of the delta with removals is checked against
              torch.searchsorted.  k_delta_adjust's and (insert-only) k_delta_count's own times come from a
              torch.profiler pass after the timed calls.
  removes     one remove of 2^16 and of 2^20 present keys from a delta of 2^20 inserted keys (host clock around the
              synchronous call; a fresh delta for every timed remove).
  compaction  merged_keys() at 200M + 2^20 - 2^20 keys (host clock), and its kernels from a torch.profiler pass: the
              merge (k_delta_merge), the subtraction (k_delta_subtract) and the sortedness check (k_check_sorted).
Per call: the median of --iters timed calls after --warmup untimed ones (CUDA events around each).  Prints one JSON
line, with the card's name and power limit read in the same run.

    python tools/delta_remove_bench.py [--keys 200000000] [--queries 134217728] [--iters 20] [--warmup 3]
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
SIZES = [(0, 1 << 16), (0, 1 << 20), (1 << 20, 1 << 20), (1 << 23, 1 << 20)]


def wrap(t):
    torch.cuda.synchronize()
    return rmi_b200.RMITrainingData.from_device(t.data_ptr(), t.numel(), rmi_b200.KEY_U64, 0, keep_alive=t)


def updated(base, keys, m, t, g):
    """A delta with m inserted and t removed keys, an insert-only delta with the same inserts (None for m == 0), and
    the logical keys, sorted, on the device."""
    n = keys.numel()
    ins = torch.sort(torch.randint(0, (1 << 63) - 1, (m,), dtype=torch.int64, device="cuda", generator=g))[0]
    from_ins = t // 2 if m else 0
    rem = torch.sort(torch.cat([keys[torch.randperm(n, device="cuda", generator=g)[: t - from_ins]],
                                ins[torch.randperm(m, device="cuda", generator=g)[:from_ins]]]))[0]
    d, only = rmi_b200.DeltaRMIIndex(base), None
    if m:
        d.insert(wrap(ins))
        only = rmi_b200.DeltaRMIIndex(base)
        only.insert(wrap(ins))
    d.remove(wrap(rem))
    M = torch.sort(torch.cat([keys, ins]))[0] if m else keys
    drop = torch.searchsorted(M, rem) + (torch.arange(t, device="cuda") - torch.searchsorted(rem, rem))
    alive = torch.ones(n + m, dtype=torch.bool, device="cuda")
    alive[drop] = False
    return d, only, M[alive]


def kernel_ms(fn, name) -> float:
    """mean milliseconds of the kernels whose name holds `name` per call of fn, from a profiled run of 5 calls"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if name in e.name]
    return round(sum(ts) / 1000.0 / 5, 4) if ts else float("nan")


def lookups(keys, base, nq, iters, warmup):
    g = torch.Generator(device="cuda")
    g.manual_seed(101)
    first = torch.empty(nq, dtype=torch.int64, device="cuda")
    last = torch.empty_like(first)
    s = torch.cuda.current_stream().cuda_stream
    out = {}
    for m, t in SIZES:
        d, only, allk = updated(base, keys, m, t, g)
        q = allk[torch.randint(0, allk.numel(), (nq,), device="cuda", generator=g)]
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
        if only is not None:
            calls["insert_only_lower_bound"] = lambda: only.lower_bound_device(p, nq, first.data_ptr(), 0, s)
            calls["insert_only_upper_bound"] = lambda: only.upper_bound_device(p, nq, last.data_ptr(), 0, s)
            calls["insert_only_equal_range"] = lambda: only.equal_range_device(p, nq, first.data_ptr(),
                                                                               last.data_ptr(), 0, s)
        e = {k: round(time_call(fn, iters, warmup), 4) for k, fn in calls.items()}
        want_lo, want_hi = torch.searchsorted(allk, q), torch.searchsorted(allk, q, right=True)
        first.fill_(-1)
        d.lower_bound_device(p, nq, first.data_ptr(), 0, s)
        exact = bool(torch.equal(first, want_lo))
        last.fill_(-1)
        d.upper_bound_device(p, nq, last.data_ptr(), 0, s)
        exact &= bool(torch.equal(last, want_hi))
        first.fill_(-1)
        last.fill_(-1)
        d.equal_range_device(p, nq, first.data_ptr(), last.data_ptr(), 0, s)
        exact &= bool(torch.equal(first, want_lo)) and bool(torch.equal(last, want_hi))
        assert exact, f"(m, t) = ({m}, {t}): an answer differs from torch.searchsorted"
        e["exact"] = exact
        e["adjust_kernel_lower_ms"] = kernel_ms(calls["delta_lower_bound"], "k_delta_adjust")
        e["adjust_kernel_equal_range_ms"] = kernel_ms(calls["delta_equal_range"], "k_delta_adjust")
        if only is not None:
            e["count_kernel_lower_ms"] = kernel_ms(calls["insert_only_lower_bound"], "k_delta_count")
            e["count_kernel_equal_range_ms"] = kernel_ms(calls["insert_only_equal_range"], "k_delta_count")
        # dependent probes per query and bound: one interleaved search over each side
        e["probes_per_query_model"] = {"inserted": math.ceil(math.log2(m + 1)), "removed": math.ceil(math.log2(t + 1))}
        out[f"{m},{t}"] = e
        d.close()
        if only is not None:
            only.close()
        del allk, q, want_lo, want_hi
        torch.cuda.empty_cache()
    return out


def removes(keys, base, reps):
    g = torch.Generator(device="cuda")
    g.manual_seed(6)
    n, m = keys.numel(), 1 << 20
    out = {}
    for b in (1 << 16, 1 << 20):
        ts = []
        for _ in range(reps):
            ins = torch.sort(torch.randint(0, (1 << 63) - 1, (m,), dtype=torch.int64, device="cuda", generator=g))[0]
            d = rmi_b200.DeltaRMIIndex(base)
            d.insert(wrap(ins))
            rem = torch.sort(torch.cat([keys[torch.randperm(n, device="cuda", generator=g)[: b // 2]],
                                        ins[torch.randperm(m, device="cuda", generator=g)[: b // 2]]]))[0]
            batch = wrap(rem)
            t0 = time.perf_counter()
            d.remove(batch)
            ts.append((time.perf_counter() - t0) * 1e3)
            d.close()
            del ins, rem, batch
        out[f"delta_{m}_remove_{b}_ms"] = round(float(np.median(ts)), 4)
    return out


def compaction(keys, base, reps):
    g = torch.Generator(device="cuda")
    g.manual_seed(78)
    n, m, t = keys.numel(), 1 << 20, 1 << 20
    d, _, allk = updated(base, keys, m, t, g)
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        merged = d.merged_keys()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
        merged.close()
    merged = d.merged_keys()
    assert len(merged) == n + m - t
    host = merged.to_numpy()
    exact = bool(np.array_equal(host.view(np.int64), allk.cpu().numpy()))
    assert exact, "merged_keys() differs from the logical keys"
    merged.close()
    res = {"merged_keys_ms": round(float(np.median(ts)), 3), "exact": exact, "keys": n + m - t}
    for k, name in (("merge_kernel_ms", "k_delta_merge"), ("subtract_kernel_ms", "k_delta_subtract"),
                    ("check_kernel_ms", "k_check_sorted")):
        res[k] = kernel_ms(lambda: d.merged_keys().close(), name)
    res["merge_bytes_model"] = 2 * (n + m) * 8
    res["subtract_bytes_model"] = (2 * (n + m) - t) * 8
    d.close()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("delta_remove_bench needs a CUDA device")
    res = {"tool": "delta_remove_bench", **gpu_info(), "spec": SPEC, "branching_factor": BF, "keys": a.keys,
           "queries": a.queries}
    keys = gen_keys("u64", a.keys)
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), a.keys, rmi_b200.KEY_U64, 0, keep_alive=keys)
    base = rmi_b200.RMIIndex(rmi_b200.train(ds, SPEC, BF, counts=False), ds)
    res["lookups"] = lookups(keys, base, a.queries, a.iters, a.warmup)
    res["removes"] = removes(keys, base, max(3, a.iters // 4))
    res["compaction"] = compaction(keys, base, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
