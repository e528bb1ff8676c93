"""The `--bounded` cache-fix spline on the device (rmi_cache_fix_device) against the host scan (rmi_cache_fix).

Workload: the headline keys of tools/bounded_lookup_bench.py (200M uniform uint64 below 2^63, generated and sorted on
the device with seed 42, key 0 dropped because cache-fix panics on it) at lines 8 and 64, plus 200M lognormal
(sigma = 2) keys scaled by 1e9 at line 8.  Per configuration:
  - the device scan: median and min seconds over --iters calls after --warmup, each a synchronous call that includes
    the copy of the knots to the host; its statistics (chunks, points, stitch segments, fallback points, spline
    evaluations) and evaluations per second;
  - train_bounded end to end on both paths: from the RMITrainingData (device scan) and from the numpy keys (host
    scan, once), with the knots asserted equal;
  - the speed-up of the scan and of train_bounded.
The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/cache_fix_bench.py [--keys 200000000] [--iters 5] [--warmup 1] [--configs uniform:8,uniform:64,lognormal:8]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import rmi_b200  # noqa: E402
from lookup_bench import gen_keys, gpu_info  # noqa: E402

SPEC, BF = "linear,linear", 1 << 20


def lognormal_keys(n: int) -> torch.Tensor:
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    z = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    k = (torch.exp(2.0 * z) * 1e9).clamp(max=float(2**62)).to(torch.int64)
    return torch.sort(k)[0]


def run(name: str, keys: torch.Tensor, line: int, iters: int, warmup: int) -> dict:
    n = keys.numel()
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=keys)
    for _ in range(warmup):
        rmi_b200.cache_fix(ds, line)
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        knots, st = rmi_b200.cache_fix(ds, line, with_stats=True)
        ts.append(time.perf_counter() - t0)
    dev_s = statistics.median(ts)
    t0 = time.perf_counter()
    r_dev, k_dev = rmi_b200.train_bounded(ds, SPEC, BF, line)
    dev_train_s = time.perf_counter() - t0
    keys_np = keys.cpu().numpy().view(np.uint64)
    t0 = time.perf_counter()
    r_host, k_host = rmi_b200.train_bounded(keys_np, SPEC, BF, line)
    host_train_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    rmi_b200.train(rmi_b200.RMITrainingData(np.ascontiguousarray(k_host[:, 0])), SPEC, BF)
    knot_rmi_s = time.perf_counter() - t0
    assert np.array_equal(knots, k_host) and np.array_equal(k_dev, k_host), "device knots differ from the host scan"
    assert r_dev.num_rmi_rows == r_host.num_rmi_rows
    host_scan_s = host_train_s - knot_rmi_s   # the RMI over the knots is the same GPU build on both paths
    ds.close()
    return {"keys": name, "line": line, "n": n, "knots": int(knots.shape[0]), "stats": st,
            "device_scan_s_median": dev_s, "device_scan_s_min": min(ts),
            "evaluations_per_s": st["evaluations"] / dev_s,
            "evaluations_per_point": st["evaluations"] / st["points"],
            "host_scan_s": host_scan_s, "scan_speedup": host_scan_s / dev_s,
            "train_bounded_device_s": dev_train_s, "train_bounded_host_s": host_train_s,
            "train_bounded_speedup": host_train_s / dev_train_s, "knots_equal": True}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="uniform:8,uniform:64,lognormal:8")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("cache_fix_bench needs a CUDA device")
    rmi_b200.load_library()
    out = {**gpu_info(), "version": rmi_b200.version(), "spec": SPEC, "branching_factor": BF, "iters": a.iters,
           "warmup": a.warmup, "results": []}
    sets = {}
    for cfg in a.configs.split(","):
        name, line = cfg.split(":")
        if name not in sets:
            k = gen_keys("u64", a.keys) if name == "uniform" else lognormal_keys(a.keys)
            sets = {name: k[k > 0].contiguous()}   # one key set resident at a time
        out["results"].append(run(name, sets[name], int(line), a.iters, a.warmup))
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
