"""rmi_b200 — H100-native two-layer RMI trainer behind the reference's `rmi_lib::train` surface.

The product is the C-ABI shared library ``rmi_b200/lib/librmi_b200.so`` (CUDA, sm_90a;
``include/rmi_b200.h``).  This package is the thin Python host side used by the tests and
``bench.py``: it mirrors the reference's public API names

    rmi_lib::train(data, model_spec, branch_factor) -> TrainedRMI      (train/mod.rs:100)
    rmi_lib::train_bounded(data, model_spec, branch_factor, line_size)  (train/mod.rs:156; cache_fix.rs:106)
    rmi_lib::train_for_size / optimizer::find_pareto_efficient_configs  (train/mod.rs:128, optimizer.rs:233)
    rmi_lib::output_rmi / rmi_size                                      (codegen.rs:757, :375)
    load_rmi (output_rmi's inverse) / evaluate (two_layer.rs:205-284 over given tables)
    RMITrainingData / load_data                                         (models/mod.rs:233, src/load.rs:132)

plus RMIIndex and BoundedRMIIndex (a train_bounded build), batched lookups (position estimates and exact lower
bounds) on the GPU.  cache_fix / train_bounded on an RMITrainingData fit the cache-fix spline on the GPU.
rmi_b200.sharded (torch.distributed) trains over range-partitioned keys (train_sharded), evaluates a given RMI over
them (evaluate_sharded) and serves lookups over them (ShardedRMIIndex).  DeltaRMIIndex serves exact lookups over keys
inserted into and removed from an index after it was built, and compacts them into a fresh index.

and does no arithmetic of its own.  There is no CPU fallback: if the CUDA library is missing
or no device is present, calls raise.
"""
from .api import (BoundedRMIIndex, DeltaRMIIndex, KEY_F64, KEY_U32, KEY_U64, FLAG_LEAF_COUNTS, FLAG_SHARD_ROOT_ONLY, FLAG_STATS_ONLY, FLAG_TOP_FIT_EXACT, RMIError, RMIIndex, RMIPanic,
                  RMITrainingData, TrainedRMI, cache_fix, evaluate, find_pareto_efficient_configs, kernel_launch_count, lib_path,
                  load_data, load_library, load_rmi, output_rmi, rmi_size, train, train_bounded, train_for_size, train_stats_batch, version)

__all__ = ["BoundedRMIIndex", "DeltaRMIIndex", "KEY_F64", "KEY_U32", "KEY_U64", "FLAG_LEAF_COUNTS", "FLAG_SHARD_ROOT_ONLY", "FLAG_STATS_ONLY", "FLAG_TOP_FIT_EXACT", "RMIError", "RMIIndex", "RMIPanic",
           "RMITrainingData", "TrainedRMI", "cache_fix", "evaluate", "find_pareto_efficient_configs", "kernel_launch_count", "lib_path",
           "load_data", "load_library", "load_rmi", "output_rmi", "rmi_size", "train", "train_bounded", "train_for_size", "train_stats_batch", "version"]
