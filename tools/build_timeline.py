"""Where a resident build's step goes: device phases against the gaps between builds and the copy tail.

  python tools/build_timeline.py [--steps K] [--warmup W] [--profile-steps P] [--out DIR]

The workload is bench.py's headline build (linear,linear 2^20 on 200M sorted uniform uint64 keys drawn with
torch.randint from a device generator seeded 42).  Two runs, in this order:

1. untraced: K back-to-back synchronous builds between two CUDA events (as bench.py times them): ms_per_step, the
   mean device_time_ns and phase_device_ns the library reports, and the mean library wall (build_time) and Python
   wall per step;
2. under torch.profiler (CUDA activities; the Chrome trace goes to DIR): per build, the GPU idle time from the end of
   the previous build's last activity to this build's first, how long the record copies (device-to-host, > 4 KiB) run
   past the end of the last k_leaf kernel, and the gaps between consecutive kernels inside the build.

Prints one JSON line, with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info():
    """(name, power limit in W or None) of the current device"""
    import torch
    name = torch.cuda.get_device_name()
    limit = None
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        limit = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                                  "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
            limit = float(out.stdout.strip().splitlines()[0])
        except Exception:
            pass
    return name, limit


def short_name(name: str) -> str:
    """a kernel's name without its template arguments and parameter list"""
    base = re.split(r"[<(]", name.replace("(anonymous namespace)", ""))[0]
    return base.split("::")[-1].split()[-1]


def analyse_trace(path: str, steps: int) -> dict:
    """Per-build idle time, record-copy tail and kernel gaps from a torch.profiler Chrome trace in which every build
    runs inside a user annotation named build_<i>."""
    with open(path) as f:
        trace = json.load(f)
    ev = trace["traceEvents"] if isinstance(trace, dict) else trace
    ranges = sorted((e["ts"], e["ts"] + e.get("dur", 0), int(e["name"].split("_")[1]))
                    for e in ev if e.get("cat") == "user_annotation" and e.get("name", "").startswith("build_"))
    launch_ts = {}   # correlation id -> host time of the runtime call that issued the GPU activity
    for e in ev:
        if e.get("cat") in ("cuda_runtime", "cuda_driver") and "correlation" in e.get("args", {}):
            launch_ts[e["args"]["correlation"]] = e["ts"]
    gpu = defaultdict(list)   # build index -> [(start, end, kind, name, bytes)]
    for e in ev:
        cat = e.get("cat")
        if cat not in ("kernel", "gpu_memcpy", "gpu_memset"):
            continue
        t = launch_ts.get(e.get("args", {}).get("correlation"))
        if t is None:
            continue
        for a, b, i in ranges:
            if a <= t <= b:
                gpu[i].append((e["ts"], e["ts"] + e["dur"], cat, e["name"], int(e.get("args", {}).get("bytes", 0))))
                break
    builds = [sorted(gpu[i]) for i in sorted(gpu)]
    idle, tails, spans, busy, d2h_after, launches = [], [], [], [], [], []
    gaps = defaultdict(list)
    prev_end = None
    for acts in builds:
        start, end = acts[0][0], max(a[1] for a in acts)
        if prev_end is not None:
            idle.append(start - prev_end)
        prev_end = end
        spans.append(end - start)
        u, cur_a, cur_b = 0.0, None, None   # union of the activities: time the GPU runs something of this build
        for a, b, *_ in acts:
            if cur_b is None or a > cur_b:
                if cur_b is not None:
                    u += cur_b - cur_a
                cur_a, cur_b = a, b
            else:
                cur_b = max(cur_b, b)
        busy.append(u + (cur_b - cur_a))
        leaf_end = max((b for a, b, c, n, _ in acts if c == "kernel" and short_name(n) == "k_leaf"), default=None)
        rec_end = max((b for a, b, c, n, by in acts if c == "gpu_memcpy" and "DtoH" in n and by > 4096), default=None)
        if leaf_end is not None and rec_end is not None:
            tails.append(rec_end - leaf_end)
        if leaf_end is not None:
            d2h_after.append(end - leaf_end)
        kern = [(a, b, short_name(n)) for a, b, c, n, _ in acts if c == "kernel"]
        launches.append(len(kern))
        reach, last = None, None
        for a, b, n in kern:
            if reach is not None:
                gaps[f"{last} -> {n}"].append(max(0.0, a - reach))
            if reach is None or b > reach:
                reach, last = b, n
    mean = lambda v: round(sum(v) / len(v), 2) if v else None
    return {"builds_traced": len(builds),
            "idle_between_builds_us": mean(idle), "idle_between_builds_us_max": round(max(idle), 2) if idle else None,
            "record_copy_past_last_k_leaf_us": mean(tails),
            "build_end_past_last_k_leaf_us": mean(d2h_after),
            "build_span_us": mean(spans), "build_gpu_busy_us": mean(busy),
            "kernels_per_build": mean(launches),
            "kernel_gaps_us": {k: mean(v) for k, v in sorted(gaps.items(), key=lambda kv: -sum(kv[1]))},
            "kernel_gaps_total_us": mean([sum(v[i] for v in gaps.values() if i < len(v)) for i in range(len(builds))])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=float, default=200e6)
    ap.add_argument("--leaves", type=int, default=1 << 20)
    ap.add_argument("--spec", default="linear,linear")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=8)
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: a new temporary one)")
    args = ap.parse_args()

    import numpy as np
    import torch
    import rmi_b200

    if not torch.cuda.is_available():
        raise SystemExit("build_timeline.py needs a CUDA device")
    rmi_b200.load_library()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out_dir = args.out or tempfile.mkdtemp(prefix="build_timeline_")
    os.makedirs(out_dir, exist_ok=True)

    n, N = int(args.keys), args.leaves
    g = torch.Generator(device=dev)
    g.manual_seed(42)
    k = torch.randint(0, (1 << 63) - 1, (n,), dtype=torch.int64, device=dev, generator=g)
    k, _ = torch.sort(k)
    torch.cuda.synchronize()
    ds = rmi_b200.RMITrainingData.from_device(k.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=k)

    def build():
        return rmi_b200.train(ds, args.spec, N, 0, counts=False)

    res = None
    for _ in range(max(args.warmup, 3)):
        res = build()
    res = None
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ns, phase, lib_wall, py_wall = 0.0, np.zeros(4), 0.0, 0.0
    e0.record()
    for _ in range(args.steps):
        t0 = time.perf_counter()
        res = build()
        py_wall += time.perf_counter() - t0
        lib_wall += res.build_time
        dev_ns += res.device_time_ns
        phase += np.array(res.phase_device_ns, dtype=np.float64)
    e1.record()
    torch.cuda.synchronize()
    K = args.steps
    ms_per_step = e0.elapsed_time(e1) / K
    timing = {"ms_per_step": round(ms_per_step, 4), "keys_per_s": n / (ms_per_step / 1e3),
              "device_time_ms": round(dev_ns / K / 1e6, 4), "phases_ms": [round(p / K / 1e6, 4) for p in phase],
              "library_wall_ms": round(lib_wall / K / 1e6, 4), "python_wall_ms": round(py_wall / K * 1e3, 4),
              "step_minus_device_ms": round(ms_per_step - dev_ns / K / 1e6, 4)}

    res = None
    from torch.profiler import ProfilerActivity, profile, record_function
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.profile_steps):
            with record_function(f"build_{i}"):
                res = build()
        torch.cuda.synchronize()
    trace = os.path.join(out_dir, "build_timeline.pt.trace.json")
    prof.export_chrome_trace(trace)
    traced = analyse_trace(trace, args.profile_steps)

    name, limit = card_info()
    print(json.dumps({"workload": f"{args.spec} {N} on {n} sorted uniform uint64 (seed 42)", "gpu": name,
                      "power_limit_w": limit, "steps": K, **timing, "trace": trace, "traced": traced}))


if __name__ == "__main__":
    main()
