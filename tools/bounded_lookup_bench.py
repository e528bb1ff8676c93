"""Batched lookups on a `--bounded` RMI (BoundedRMIIndex) against the plain RMIIndex and torch.searchsorted.

Workload: the headline keys of tools/lookup_bench.py (200M uniform uint64 below 2^63, generated and sorted on the
device with the same seed, key 0 dropped because cache-fix panics on it); per line size (--lines, default 8,64) the
host cache-fix scan, `linear,linear 2^20` over its knots, and the three query sets of lookup_bench.py (2^27 random
present keys, the same sorted, uniform over [min, max]).  Line 8 gives about n/8.5 knots (~380 MB, far above the
50 MB L2) and line 64 about n/64 (~50 MB, about the L2), so the two lines sit on both sides of L2 residency, and on
both sides of the kernel's choice between counting a line's keys (line <= 16) and binary-searching it.

Per query set: bounded predict and lower_bound (median ms over --iters CUDA-event-timed calls after --warmup, Gq/s,
fallbacks, equality with torch.searchsorted), the plain index over all keys (same spec) and torch.searchsorted on
the same queries, the speed-ups, and a per-query sector model computed from shapes (32-byte sectors: the knot RMI's
leaf record, ceil(log2(2e+1)) knot probes over the knot window, the two adjacent knot records, the key line as the
kernel reads it, and the edge probes it issues).  Prints one JSON line.

    python tools/bounded_lookup_bench.py [--keys 200000000] [--queries 134217728] [--lines 8,64] [--iters 20]
"""
from __future__ import annotations

import argparse
import json
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
COUNT_MAX = 16   # kernels_lookup.cu BOUNDED_COUNT_MAX: longer lines are binary-searched


def sector_model(line: int, n: int, knot_err: torch.Tensor, pos: torch.Tensor, lb: torch.Tensor) -> dict:
    """Mean 32-byte sectors per bounded lower_bound, from the knot windows, predictions and answers."""
    knot_probes = float(torch.ceil(torch.log2(2.0 * knot_err.double() + 1.0)).mean())
    lo = torch.clamp(pos, max=n)
    hi = torch.clamp(lo + line, max=n)
    if line <= COUNT_MAX:   # every key of [lo, hi) is loaded
        span = torch.where(hi > lo, (8 * hi - 1) // 32 - (8 * lo) // 32 + 1, torch.zeros_like(lo))
        key_sectors = float(span.double().mean())
    else:                   # branchless binary search: ceil(log2(len)) + 1 probes
        key_sectors = float(torch.ceil(torch.log2((hi - lo).clamp(min=1).double())).mean()) + 1.0
    left = ((lb == lo) & (lo > 0)).double().mean()
    right = ((lb >= hi) & (hi < n)).double().mean()
    edge = float(left + right)
    total = 1.0 + knot_probes + 1.5 + key_sectors + edge
    return {"leaf_record": 1, "knot_probes": round(knot_probes, 2), "knot_record_sectors": 1.5,
            "key_line_sectors": round(key_sectors, 2), "edge_probes": round(edge, 3),
            "total_sectors": round(total, 2), "random_bytes": round(32.0 * total, 1)}


def run_line(keys, keys_np, line, plain, qsets, iters, warmup):
    n = keys.numel()
    t0 = time.perf_counter()
    knots = rmi_b200.cache_fix(keys_np, line)
    cache_fix_s = time.perf_counter() - t0
    kds = rmi_b200.RMITrainingData(np.ascontiguousarray(knots[:, 0]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = rmi_b200.train(kds, SPEC, BF, counts=False)
    train_s = time.perf_counter() - t0
    r.num_data_rows = n
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=keys)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx = rmi_b200.BoundedRMIIndex(r, knots, line, ds)
    torch.cuda.synchronize()
    create_ms = (time.perf_counter() - t0) * 1e3
    over_knots = rmi_b200.RMIIndex(r, kds)     # for the knot windows of the sector model
    nq = next(iter(qsets.values())).numel()
    pos = torch.empty(nq, dtype=torch.int64, device="cuda")
    err = torch.empty_like(pos)
    out = torch.empty_like(pos)
    fb = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    res = {"line_size": line, "knots": int(knots.shape[0]), "knot_bytes": int(knots.nbytes),
           "cache_fix_s": round(cache_fix_s, 2), "train_s": round(train_s, 3), "index_create_ms": round(create_ms, 2),
           "queries": {}}
    for qname, q in qsets.items():
        ms_p = time_call(lambda: idx.predict_device(q.data_ptr(), nq, pos.data_ptr(), err.data_ptr(), s), iters, warmup)
        ms_l = time_call(lambda: idx.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), 0, s), iters, warmup)
        ms_plain = time_call(lambda: plain.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), 0, s), iters, warmup)
        ms_s = time_call(lambda: torch.searchsorted(keys, q), iters, warmup)
        fb.zero_()
        idx.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), fb.data_ptr(), s)
        want = torch.searchsorted(keys, q)
        ok = bool(torch.equal(out, want))
        idx.predict_device(q.data_ptr(), nq, pos.data_ptr(), 0, s)
        over_knots.predict_device(q.data_ptr(), nq, out.data_ptr(), err.data_ptr(), s)
        model = sector_model(line, n, err, pos, want)
        del want
        res["queries"][qname] = {
            "bounded_predict": {"ms": round(ms_p, 4), "gq_per_s": round(nq / ms_p / 1e6, 3)},
            "bounded_lower_bound": {"ms": round(ms_l, 4), "gq_per_s": round(nq / ms_l / 1e6, 3)},
            "plain_lower_bound": {"ms": round(ms_plain, 4), "gq_per_s": round(nq / ms_plain / 1e6, 3)},
            "searchsorted": {"ms": round(ms_s, 4), "gq_per_s": round(nq / ms_s / 1e6, 3)},
            "fallbacks": int(fb.item()), "lower_bound_equals_searchsorted": ok,
            "speedup_vs_plain": round(ms_plain / ms_l, 3), "speedup_vs_searchsorted": round(ms_s / ms_l, 3),
            "mean_knot_err": round(float(err.double().mean()), 2), "sector_model": model}
    idx.close()
    over_knots.close()
    kds.close()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27)
    ap.add_argument("--lines", default="8,64")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bounded_lookup_bench needs a CUDA device")
    rmi_b200.load_library()
    info = gpu_info()
    keys = gen_keys("u64", a.keys)
    keys = keys[keys > 0].contiguous()
    n = keys.numel()
    keys_np = keys.cpu().numpy().view(np.uint64)
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=keys)
    plain = rmi_b200.RMIIndex(rmi_b200.train(ds, SPEC, BF, counts=False), ds)
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    present = keys[torch.randint(0, n, (a.queries,), device="cuda", generator=g)]
    qsets = {"present_random": present, "present_sorted": torch.sort(present)[0],
             "uniform": torch.randint(int(keys[0]), int(keys[-1]) + 1, (a.queries,), dtype=keys.dtype, device="cuda",
                                      generator=g)}
    out = {**info, "version": rmi_b200.version(), "spec": SPEC, "branching_factor": BF, "keys": n,
           "queries": a.queries, "iters": a.iters, "warmup": a.warmup,
           "results": [run_line(keys, keys_np, int(line), plain, qsets, a.iters, a.warmup)
                       for line in a.lines.split(",")]}
    plain.close()
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
