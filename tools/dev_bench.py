"""Developer timing probe (not the contract bench): per-phase device times at full size."""
import sys, os, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import rmi_b200

pos = [a for a in sys.argv[1:] if not a.startswith("--")]
opt = {a.split("=")[0]: (a.split("=") + ["1"])[1] for a in sys.argv[1:] if a.startswith("--")}
n = int(float(pos[0])) if pos else 200_000_000
torch.manual_seed(int(opt.get("--seed", 42)))
dev = torch.device("cuda:0")
k = torch.randint(0, (2**63 - 1) // int(opt.get("--div", 1)), (n,), dtype=torch.int64, device=dev)
k, _ = torch.sort(k)
torch.cuda.synchronize()
ds = rmi_b200.RMITrainingData.from_device(k.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=k)
configs = [("linear,linear", 1 << 20, 0), ("radix,linear", 1 << 19, 0), ("cubic,linear", 1 << 18, 0),
           ("linear,linear", 1 << 20, rmi_b200.FLAG_STATS_ONLY), ("linear_spline,cubic", 1 << 18, 0),
           ("radix18,linear", 1 << 16, 0), ("bradix,linear", 1 << 18, 0), ("histogram,linear", 1 << 16, 0)]
if "--quick" in opt:
    configs = configs[:3]
if "--long" in opt:   # long training vectors: what each GPU of an 8-GPU sharded build sees (1525 keys per leaf), and beyond
    configs = [("linear,linear", 1 << 20, 0), ("linear,linear", 1 << 18, 0), ("linear,linear", 1 << 17, 0),
               ("linear,linear", 1 << 14, 0), ("cubic,linear", 1 << 18, 0), ("linear,cubic", 1 << 17, 0)]
if "--spec" in opt:
    configs = [(opt["--spec"], int(opt.get("--bf", 1 << 20)), 0)]
if "--one" in opt:
    configs = configs[:1]
if "--exact" in opt:
    configs.append(("linear,linear", 1 << 20, rmi_b200.FLAG_TOP_FIT_EXACT))
for spec, bf, flags in configs:
    try:
        walls, devs, leafs = [], [], []
        for it in range(int(opt.get("--iters", 3))):
            t0 = time.perf_counter()
            r = rmi_b200.train(ds, spec, bf, flags, counts="--counts" in opt)
            t1 = time.perf_counter()
            walls.append((t1 - t0) * 1e3); devs.append(r.device_time_ns / 1e6); leafs.append(r.phase_device_ns[2] / 1e6)
        walls.sort(); devs.sort(); leafs.sort()
        print(json.dumps({"spec": spec, "bf": bf, "flags": flags, "wall_ms": (t1 - t0) * 1e3,
                          "wall_ms_min": walls[0], "wall_ms_med": walls[len(walls) // 2], "device_ms_min": devs[0],
                          "leaf_ms_min": leafs[0], "leaf_ms_med": leafs[len(leafs) // 2],
                          "lib_wall_ms": r.build_time / 1e6, "device_ms": r.device_time_ns / 1e6,
                          "phases_ms": [p / 1e6 for p in r.phase_device_ns], "max_err": r.model_max_error, "max_leaf_keys": int(r.l1_counts.max()) if r.l1_counts is not None else None,
                          "avg_log2": r.model_avg_log2_error, "keys_per_s_device": n / (r.device_time_ns / 1e9)}))
    except rmi_b200.RMIError as e:
        print(json.dumps({"spec": spec, "bf": bf, "error": str(e)}))
    sys.stdout.flush()
