"""Batched lookup throughput on the GPU: RMIIndex.predict / lower_bound against torch.searchsorted.

Workloads (keys generated and sorted on the device with bench.py's seeded generator):
  linear,linear 1048576  on 200M uniform uint64 keys below 2^63  (the headline build)
  cubic,linear 262144    on the same keys
  radix,linear 524288    on 200M uniform uint32 keys below 2^31
Query sets (2^27 each): random present keys, the same keys sorted, uniform (almost always absent) keys over
[min, max].  Per call: median kernel time over --iters timed calls after --warmup untimed ones (CUDA events),
G queries/s, fallbacks, mean leaf error of the queried leaves, and a memory-traffic model computed from shapes and
errors (DRAM sectors of 32 B per query: the streamed queries and results, one leaf record (two for cubic), about
ceil(log2(2 err + 1)) dependent key probes plus 2 edge probes).  Prints one JSON line.

    python tools/lookup_bench.py [--keys 200000000] [--queries 134217728] [--iters 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rmi_b200  # noqa: E402

SPECS = [("u64", "linear,linear", 1 << 20), ("u64", "cubic,linear", 262144), ("u32", "radix,linear", 524288)]


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the measurement itself does not depend on it
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def gen_keys(kind: str, n: int):
    g = torch.Generator(device="cuda")
    if kind == "u64":
        g.manual_seed(42)
        k = torch.randint(0, (1 << 63) - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    else:
        g.manual_seed(7)
        k = torch.randint(0, (1 << 31) - 1, (n,), dtype=torch.int32, device="cuda", generator=g)
    return torch.sort(k)[0]


def time_call(fn, iters: int, warmup: int) -> float:
    """median milliseconds of fn() over `iters` calls, each bracketed by CUDA events"""
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
    return float(np.median(ts))


def traffic_model(kb: int, err: torch.Tensor, rec_sectors: int, mode: str) -> dict:
    """sectors and bytes per query from shapes and the queried leaves' error bounds"""
    stream = kb + 8 + (8 if mode == "predict" else 0)
    probes = 0.0
    if mode == "lower_bound":
        probes = float(torch.ceil(torch.log2(2.0 * err.double() + 1.0)).mean()) + 2.0
    if mode == "searchsorted":
        return {"streamed_bytes": kb + 8}
    return {"streamed_bytes": stream, "record_sectors": rec_sectors, "key_probe_sectors": round(probes, 2),
            "random_bytes": round(32.0 * (rec_sectors + probes), 1)}


def run_spec(kind, spec, bf, n, nq, iters, warmup):
    keys = gen_keys(kind, n)
    kt = rmi_b200.KEY_U64 if kind == "u64" else rmi_b200.KEY_U32
    kb = 8 if kind == "u64" else 4
    ds = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, kt, 0, keep_alive=keys)
    r = rmi_b200.train(ds, spec, bf, counts=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx = rmi_b200.RMIIndex(r, ds)
    torch.cuda.synchronize()
    create_ms = (time.perf_counter() - t0) * 1e3
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    present = keys[torch.randint(0, n, (nq,), device="cuda", generator=g)]
    qsets = {"present_random": present, "present_sorted": torch.sort(present)[0],
             "uniform": torch.randint(int(keys[0]), int(keys[-1]) + 1, (nq,), dtype=keys.dtype, device="cuda",
                                      generator=g)}
    pos = torch.empty(nq, dtype=torch.int64, device="cuda")
    err = torch.empty(nq, dtype=torch.int64, device="cuda")
    out = torch.empty(nq, dtype=torch.int64, device="cuda")
    fb = torch.zeros(1, dtype=torch.int64, device="cuda")
    rec_sectors = 2 if spec.split(",")[1] == "cubic" else 1
    res = {"spec": spec, "keys": n, "key_type": kind, "branching_factor": bf, "index_create_ms": round(create_ms, 2),
           "record_bytes": 32 * rec_sectors, "queries": {}}
    for qname, q in qsets.items():
        s = torch.cuda.current_stream().cuda_stream
        ms_p = time_call(lambda: idx.predict_device(q.data_ptr(), nq, pos.data_ptr(), err.data_ptr(), s), iters, warmup)
        ms_l = time_call(lambda: idx.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), 0, s), iters, warmup)
        ms_s = time_call(lambda: torch.searchsorted(keys, q), iters, warmup)
        fb.zero_()
        idx.lower_bound_device(q.data_ptr(), nq, out.data_ptr(), fb.data_ptr(), s)
        ok = bool(torch.equal(out, torch.searchsorted(keys, q)))
        mean_err = float(err.double().mean())
        e = {}
        for mode, ms in (("predict", ms_p), ("lower_bound", ms_l), ("searchsorted", ms_s)):
            e[mode] = {"ms": round(ms, 4), "gq_per_s": round(nq / ms / 1e6, 3), **traffic_model(kb, err, rec_sectors, mode)}
        e["fallbacks"] = int(fb.item())
        e["mean_leaf_err"] = round(mean_err, 2)
        e["lower_bound_equals_searchsorted"] = ok
        e["lower_bound_speedup_vs_searchsorted"] = round(ms_s / ms_l, 3)
        res["queries"][qname] = e
    idx.close()
    del ds, keys
    torch.cuda.empty_cache()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--queries", type=int, default=1 << 27)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--specs", default="all", help="'all' or a comma-separated list of indices into the workload list")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("lookup_bench needs a CUDA device")
    rmi_b200.load_library()
    specs = SPECS if a.specs == "all" else [SPECS[int(i)] for i in a.specs.split(",")]
    out = {**gpu_info(), "version": rmi_b200.version(), "iters": a.iters, "warmup": a.warmup,
           "results": [run_spec(k, s, bf, a.keys, a.queries, a.iters, a.warmup) for k, s, bf in specs]}
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
