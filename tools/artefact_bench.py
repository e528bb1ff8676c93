"""rmi_evaluate against rmi_train, and the artefact round trip, on the headline workload.

Workload: 200M uniform uint64 keys below 2^63 (generated and sorted on the device with bench.py's seeded generator),
linear,linear with 2^20 leaves.  After --warmup untimed calls of each, --iters timed calls of
  train     rmi_train (with leaf counts)                      wall time, device time, phases
  evaluate  rmi_evaluate of the trained tables on the same keys wall time, device time, phases
            ([0] table upload, [1] leaf boundaries, [2] error pass, [3] statistics)
and the medians are reported.  The error pass's algorithmic traffic is 8n bytes of keys plus, per leaf, its
parameters, two boundaries and the error and count it writes; over the pass's CUDA-event time (phase [2]) it is
given as a fraction of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s.  output_rmi / load_rmi of the 2^20-leaf
artefact (a 24 MB blob) are timed in a temporary directory.  The card's name and power limit are read in the same
call.  Prints one JSON line.

    python tools/artefact_bench.py [--keys 200000000] [--iters 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import rmi_b200  # noqa: E402
from lookup_bench import gen_keys, gpu_info  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def timed(fn, iters: int, warmup: int):
    for _ in range(warmup):
        fn()
    runs = []
    for _ in range(iters):
        t0 = time.perf_counter()
        r = fn()
        runs.append((time.perf_counter() - t0, r))
    wall = statistics.median(w for w, _ in runs)
    dev = statistics.median(r.device_time_ns for _, r in runs)
    phases = [statistics.median(r.phase_device_ns[q] for _, r in runs) for q in range(4)]
    return wall, dev, phases, runs[-1][1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--leaves", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    info = gpu_info()
    k = gen_keys("u64", a.keys)
    torch.cuda.synchronize()
    ds = rmi_b200.RMITrainingData.from_device(k.data_ptr(), a.keys, rmi_b200.KEY_U64, 0, keep_alive=k)
    spec, N = "linear,linear", a.leaves
    t_wall, t_dev, t_ph, g = timed(lambda: rmi_b200.train(ds, spec, N), a.iters, a.warmup)
    e_wall, e_dev, e_ph, e = timed(lambda: rmi_b200.evaluate(g, ds), a.iters, a.warmup)
    same = bool(np.array_equal(e.last_layer_max_l1s, g.last_layer_max_l1s) and np.array_equal(e.l1_counts, g.l1_counts))
    ppm = g.l1_params.shape[1]
    pass_bytes = 8 * a.keys + N * (8 * ppm + 2 * 8 + 2 * 8)
    pass_s = e_ph[2] / 1e9
    with tempfile.TemporaryDirectory() as d:
        data_dir = os.path.join(d, "rmi_data")
        t0 = time.perf_counter()
        rmi_b200.output_rmi("rmi", g, data_dir, out_dir=d)
        out_s = time.perf_counter() - t0
        blob = os.path.getsize(os.path.join(data_dir, "rmi_L1_PARAMETERS"))
        t0 = time.perf_counter()
        loaded, _ = rmi_b200.load_rmi("rmi", d, data_dir)
        load_s = time.perf_counter() - t0
        loaded_ok = bool(np.array_equal(loaded.l1_params.view(np.uint64), g.l1_params.view(np.uint64)))
    print(json.dumps({
        **info, "keys": a.keys, "spec": spec, "leaves": N, "iters": a.iters,
        "train": {"wall_ms": t_wall * 1e3, "device_ms": t_dev / 1e6, "phases_ms": [p / 1e6 for p in t_ph]},
        "evaluate": {"wall_ms": e_wall * 1e3, "device_ms": e_dev / 1e6, "phases_ms": [p / 1e6 for p in e_ph]},
        "evaluate_equals_train": same,
        "error_pass": {"bytes": pass_bytes, "ms": pass_s * 1e3, "GB_per_s": pass_bytes / pass_s / 1e9,
                       "fraction_of_3.35TBps": pass_bytes / pass_s / PEAK_BYTES_PER_S},
        "artefact": {"blob_bytes": blob, "output_rmi_ms": out_s * 1e3, "load_rmi_ms": load_s * 1e3, "loaded_equal": loaded_ok},
    }))


if __name__ == "__main__":
    main()
