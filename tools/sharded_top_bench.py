"""The bradix and loglinear top models over range-partitioned keys: train_sharded's one-call form (rmi_shard_train,
a one-rank NCCL communicator) against rmi_train of the same keys on one GPU, in the same run.

Workload: 200M uniform uint64 keys below 2^63 (bench.py's seeded generator), bradix,linear and loglinear,linear at
2^20 leaves.  Per spec: median of --iters builds after --warmup untimed ones, per phase of the result's
phase_device_ns (CUDA events: top fit, leaf boundaries, leaf fit + error pass, statistics).  The sharded top fit of
bradix counts the keys of all four candidates in one pass; rmi_train's reads the keys once per candidate.  Asserts
the rules the tests hold the two to: bradix bit for bit; loglinear's top within 1e-9 (relative to its terms, the
intercept to ln(N)), and rmi_train given that top bit for bit.  Prints one JSON line.

    python tools/sharded_top_bench.py
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rmi_b200  # noqa: E402
from rmi_b200 import sharded  # noqa: E402
from tools.sharded_lookup_bench import gpu_info  # noqa: E402

PHASES = ("top", "boundaries", "leaves", "statistics")


def bits(v):
    return np.asarray(v, dtype=np.float64).view(np.uint64)


def same(a, b) -> bool:
    return (np.array_equal(bits(a.l0_fparams), bits(b.l0_fparams)) and np.array_equal(a.l0_iparams, b.l0_iparams)
            and a.l0_bradix_high == b.l0_bradix_high and np.array_equal(bits(a.l1_params), bits(b.l1_params))
            and np.array_equal(a.last_layer_max_l1s, b.last_layer_max_l1s)
            and (a.model_max_error, a.model_max_error_idx, a.model_avg_error) ==
            (b.model_max_error, b.model_max_error_idx, b.model_avg_error))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=200_000_000)
    ap.add_argument("--leaves", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("sharded_top_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, N = a.keys, a.leaves
    g = torch.Generator(device=dev)
    g.manual_seed(42)
    keys = torch.sort(torch.randint(0, (1 << 63) - 1, (n,), dtype=torch.int64, device=dev, generator=g))[0]
    full = rmi_b200.RMITrainingData.from_device(keys.data_ptr(), n, rmi_b200.KEY_U64, dev.index, keep_alive=keys)
    data = sharded.ShardedTrainingData(keys.clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
    if sharded.native_comm(None, dev, single_rank_ok=True) is None:
        raise SystemExit("the one-call form needs NCCL (libnccl.so.2)")

    def run(fn):
        for _ in range(a.warmup):
            fn()
        phases, last = [], None
        for _ in range(a.iters):
            last = fn()
            phases.append(list(last.phase_device_ns))
        return {p: round(float(np.median([r[q] for r in phases])) / 1e6, 4) for q, p in enumerate(PHASES)}, last

    out = {"world": 1, "keys": n, "branching_factor": N, "iters": a.iters, "warmup": a.warmup,
           "version": rmi_b200.version()}
    equal = True
    for spec in ("bradix,linear", "loglinear,linear"):
        s_ms, s = run(lambda: sharded.train_sharded(data, spec, N, native=True, counts=False))
        t_ms, t = run(lambda: rmi_b200.train(full, spec, N, counts=False))
        top = spec.split(",")[0]
        if top == "loglinear":
            rel = np.abs(s.l0_fparams - t.l0_fparams) / np.maximum(np.abs(t.l0_fparams), [np.log(N), 0.0])
            ok = bool((rel <= 1e-9).all()) and same(s, rmi_b200.train(full, spec, N, l0_params=s.l0_fparams, counts=False))
            out[f"{top}_top_rel_err"] = [float(x) for x in rel]
        else:
            ok = same(s, t)
        equal = equal and ok
        out[f"{top}_sharded_phase_ms"] = s_ms
        out[f"{top}_rmi_train_phase_ms"] = t_ms
    out["equal"] = equal
    print(json.dumps({**gpu_info(), **out}))
    if not equal:
        raise SystemExit("the sharded build differs from rmi_train")
    return out


if __name__ == "__main__":
    main()
