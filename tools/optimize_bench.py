"""BASELINE.json configs[4]: the `--optimize` sweep (optimizer.rs:110-151, :220-249) on 800M synthetic f64 keys over the
GPUs of one node, measured; plus the parity of the search itself on a sample the CPU oracle can sweep.

    python tools/optimize_bench.py [--keys 800e6] [--gpus 8] [--sample 4e6] > optimize_<N>gpu.json

One process: the keys are generated and sorted on GPU 0, replicated to the other GPUs over NVLink
(rmi_dataset_replicate), and rmi_find_pareto_efficient_configs spreads the (top, branching factor) groups over one
host thread per replica.  Reported: seconds and configurations/s for 1 and N replicas, with and without the per-group
batching (rmi_train_stats_batch), the resulting front, and — on a `--sample`-key prefix-stride sample — the GPU sweep's
per-configuration statistics and front against the same search driven by the CPU oracle."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=float, default=800e6)
    ap.add_argument("--gpus", type=int, default=0, help="0 = all visible")
    ap.add_argument("--sample", type=float, default=4e6)
    ap.add_argument("--dist", default="uniform", choices=["uniform", "lognormal"])
    ap.add_argument("--skip-single", action="store_true", help="do not time the one-replica sweep as well")
    args = ap.parse_args()
    import numpy as np
    import torch
    import rmi_b200
    from tests import test_optimizer as topt

    n = int(args.keys)
    ngpu = args.gpus or torch.cuda.device_count()
    dev0 = torch.device("cuda", 0)
    g = torch.Generator(device=dev0)
    g.manual_seed(11)
    if args.dist == "uniform":      # SURVEY 8(d) config 5: sorted uniform(0, 2^52) doubles, seed 11
        k = torch.rand(n, dtype=torch.float64, device=dev0, generator=g) * float(1 << 52)
    else:
        k = torch.exp(torch.randn(n, dtype=torch.float64, device=dev0, generator=g) * 2.0)
    k, _ = torch.sort(k)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ds0 = rmi_b200.RMITrainingData.from_device(k.data_ptr(), n, rmi_b200.KEY_F64, 0, keep_alive=k)
    reps = [ds0] + [ds0.replicate(d) for d in range(1, ngpu)]
    t_rep = time.perf_counter() - t0
    out = {"keys": n, "key_type": "f64", "distribution": args.dist, "gpus": ngpu, "replicate_seconds": t_rep,
           "profile": os.environ.get("RMI_OPTIMIZER_PROFILE", "(default: memory)")}

    def sweep(replicas, label):
        launches0 = rmi_b200.kernel_launch_count()
        t0 = time.perf_counter()
        front = rmi_b200.find_pareto_efficient_configs(replicas, 10)
        dt = time.perf_counter() - t0
        out[label] = {"seconds": dt, "kernel_launches": rmi_b200.kernel_launch_count() - launches0, "front": front}
        return front

    # number of configurations of the two phases (the second phase depends on the first's results: recount from the grid)
    first = topt.first_phase("")
    out["phase1_configs"] = len(first)
    f_n = sweep(reps, f"sweep_{ngpu}_replicas_batched")
    if ngpu > 1 and not args.skip_single:
        sweep(reps[:1], "sweep_1_replica_batched")
    os.environ["RMI_OPTIMIZER_NO_BATCH"] = "1"   # read once per process by the library: only effective in a fresh process
    out["note_unbatched"] = "the unbatched sweep is timed by a second invocation with RMI_OPTIMIZER_NO_BATCH=1 (see *_nobatch.json)"
    out["front_models"] = [(c["models"], c["branching_factor"]) for c in f_n]

    # ---- parity of the search on a sample the oracle can sweep --------------------------------------------------
    ns = int(args.sample)
    if ns > 0:
        import oracle
        oracle.build()
        ks = k[:: max(n // ns, 1)][:ns].contiguous()
        host = ks.cpu().numpy()
        dss = rmi_b200.RMITrainingData.from_device(ks.data_ptr(), host.size, rmi_b200.KEY_F64, 0, keep_alive=ks)
        tops = {}
        gpu_stats, cpu_stats, mism = [], [], []
        t0 = time.perf_counter()
        for spec, bf in first:
            top, leaf = spec.split(",")
            r = rmi_b200.train(dss, spec, bf, rmi_b200.FLAG_STATS_ONLY, counts=False)
            gpu_stats.append((spec, bf, r.model_avg_log2_error, r.model_max_log2_error, rmi_b200.rmi_size(r)))
        t_gpu = time.perf_counter() - t0
        t0 = time.perf_counter()
        for (spec, bf), gs in zip(first, gpu_stats):
            top = spec.split(",")[0]
            # tops with an order-dependent float fit: compare given the GPU's top coefficients (tests/parity.py rules)
            l0 = None
            if top in ("robust_linear", "linear", "cubic"):
                l0 = rmi_b200.train(dss, spec, bf, rmi_b200.FLAG_STATS_ONLY, counts=False).l0_fparams
            o = oracle.train(host, spec, bf, l0_override=l0)
            size = gs[4]
            cpu_stats.append((spec, bf, o.avg_log2_error, o.max_log2_error, size))
            if abs(o.avg_log2_error - gs[2]) > 1e-10 * max(abs(o.avg_log2_error), 1e-300) or o.max_log2_error != gs[3]:
                mism.append((spec, bf, gs[2], o.avg_log2_error, gs[3], o.max_log2_error))
        t_cpu = time.perf_counter() - t0
        same_front = ([(x[0], x[1]) for x in topt.pareto(gpu_stats)] == [(x[0], x[1]) for x in topt.pareto(cpu_stats)])
        out["sample_parity"] = {"sample_keys": int(host.size), "configs": len(first), "gpu_seconds": t_gpu, "oracle_seconds": t_cpu,
                                "stat_mismatches": mism[:10], "n_mismatches": len(mism), "phase1_pareto_front_equal": bool(same_front)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
