"""ctypes binding of include/rmi_b200.h, shaped like the reference's Rust API."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "librmi_b200.so")

KEY_U64, KEY_U32, KEY_F64 = 0, 1, 2
FLAG_STATS_ONLY, FLAG_TOP_FIT_EXACT, FLAG_LEAF_COUNTS, FLAG_SHARD_ROOT_ONLY = 1, 2, 8, 16
_NP_OF_KEY = {KEY_U64: np.uint64, KEY_U32: np.uint32, KEY_F64: np.float64}
MODEL_NAMES = ["linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal", "radix",
               "radix_table", "bradix", "histogram"]


class RMIError(RuntimeError):
    """A failure at the C-ABI boundary (bad argument, CUDA error, unsupported request)."""


class RMIPanic(RMIError):
    """The reference would have panicked on this input (assert!/unwrap/panic!)."""


class _Result(C.Structure):
    """struct rmi_result (include/rmi_b200.h), mirror of TrainedRMI (train/mod.rs:18-33)."""
    _fields_ = [
        ("num_rmi_rows", C.c_uint64), ("num_data_rows", C.c_uint64), ("branching_factor", C.c_uint64),
        ("model_avg_error", C.c_double), ("model_avg_l2_error", C.c_double), ("model_avg_log2_error", C.c_double),
        ("model_max_log2_error", C.c_double), ("model_max_error", C.c_uint64), ("model_max_error_idx", C.c_uint64),
        ("build_time_ns", C.c_uint64), ("device_time_ns", C.c_uint64), ("phase_device_ns", C.c_uint64 * 4),
        ("l0_model_id", C.c_uint32), ("l0_bradix_high", C.c_uint32), ("l0_table_bits", C.c_uint32),
        ("l0_num_fparams", C.c_uint32), ("l0_fparams", C.c_double * 4), ("l0_num_iparams", C.c_uint32),
        ("_pad0", C.c_uint32), ("l0_iparams", C.c_uint64 * 4),
        ("l0_table32_len", C.c_uint64), ("l0_table32", C.POINTER(C.c_uint32)),
        ("l0_array1_len", C.c_uint64), ("l0_array1", C.POINTER(C.c_uint64)),
        ("l0_array2_len", C.c_uint64), ("l0_array2", C.POINTER(C.c_uint64)),
        ("l1_model_id", C.c_uint32), ("l1_params_per_model", C.c_uint32),
        ("l1_params", C.POINTER(C.c_double)), ("l1_errors", C.POINTER(C.c_uint64)),
        ("l1_counts", C.POINTER(C.c_uint64)), ("could_not_replace", C.c_uint32), ("top_fit_exact", C.c_uint32),
    ]


class _CacheFixStats(C.Structure):
    """struct rmi_cache_fix_stats (include/rmi_b200.h): what a device cache-fix scan did."""
    _fields_ = [("chunk_keys", C.c_uint64), ("chunks", C.c_uint64), ("points", C.c_uint64),
                ("stitch_segments", C.c_uint64), ("fallback_points", C.c_uint64), ("evaluations", C.c_uint64)]


class _ArtefactInfo(C.Structure):
    """struct rmi_artefact_info (include/rmi_b200.h): what rmi_load_rmi found besides the model."""
    _fields_ = [("key_type", C.c_int), ("has_errors", C.c_int), ("line_size", C.c_uint64), ("num_knots", C.c_uint64),
                ("num_data_rows", C.c_uint64), ("build_time_ns", C.c_uint64)]


class _ConfigStats(C.Structure):
    """struct rmi_config_stats (optimizer.rs:153-160 RMIStatistics)."""
    _fields_ = [("models", C.c_char * 64), ("branching_factor", C.c_uint64), ("average_log2_error", C.c_double),
                ("max_log2_error", C.c_double), ("size", C.c_uint64)]


_lib = None


def lib_path() -> str:
    return _LIB_PATH


def load_library():
    """Load librmi_b200.so (built in-tree by rmi_b200.build / __graft_entry__.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise RMIError(f"{_LIB_PATH} is missing: run `python -m rmi_b200.build` (there is no CPU fallback)")
        L = C.CDLL(_LIB_PATH)
        L.rmi_last_error.restype = C.c_char_p
        L.rmi_version.restype = C.c_char_p
        L.rmi_kernel_launch_count.restype = C.c_uint64
        L.rmi_dataset_create.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.rmi_dataset_wrap_device.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.rmi_dataset_load_file.argtypes = [C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.rmi_dataset_replicate.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.rmi_dataset_len.restype = C.c_uint64
        L.rmi_dataset_len.argtypes = [C.c_void_p]
        L.rmi_dataset_key_type.argtypes = [C.c_void_p]
        L.rmi_dataset_copy_to_host.argtypes = [C.c_void_p, C.c_void_p]
        L.rmi_dataset_destroy.argtypes = [C.c_void_p]
        L.rmi_train.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint32, C.POINTER(C.POINTER(_Result))]
        L.rmi_train_with_top.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32,
                                         C.POINTER(C.POINTER(_Result))]
        L.rmi_result_free.argtypes = [C.POINTER(_Result)]
        L.rmi_cache_fix.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.rmi_cache_fix_device.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                                           C.POINTER(_CacheFixStats)]
        L.rmi_spline_free.argtypes = [C.c_void_p]
        L.rmi_model_size.restype = C.c_uint64
        L.rmi_model_size.argtypes = [C.POINTER(_Result), C.c_int, C.c_uint64]
        L.rmi_output_rmi.argtypes = [C.c_char_p, C.POINTER(_Result), C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_uint64,
                                     C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
        L.rmi_load_rmi.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.POINTER(_Result)), C.POINTER(C.c_void_p),
                                   C.POINTER(_ArtefactInfo)]
        L.rmi_evaluate.argtypes = [C.c_void_p, C.POINTER(_Result), C.c_uint32, C.POINTER(C.POINTER(_Result))]
        L.rmi_find_pareto_efficient_configs.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint64, C.c_uint32,
                                                        C.POINTER(_ConfigStats), C.c_uint64, C.POINTER(C.c_uint64)]
        L.rmi_index_create.argtypes = [C.POINTER(_Result), C.c_void_p, C.POINTER(C.c_void_p)]
        L.rmi_index_create_bounded.argtypes = [C.POINTER(_Result), C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p,
                                               C.POINTER(C.c_void_p)]
        L.rmi_index_destroy.argtypes = [C.c_void_p]
        L.rmi_index_predict.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_index_lower_bound.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_index_lookup_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
        L.rmi_index_upper_bound.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_index_equal_range.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
        L.rmi_index_range_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_delta_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.rmi_delta_destroy.argtypes = [C.c_void_p]
        L.rmi_delta_insert.argtypes = [C.c_void_p, C.c_void_p]
        L.rmi_delta_len.restype = C.c_uint64
        L.rmi_delta_len.argtypes = [C.c_void_p]
        L.rmi_delta_remove.argtypes = [C.c_void_p, C.c_void_p]
        L.rmi_delta_removed_len.restype = C.c_uint64
        L.rmi_delta_removed_len.argtypes = [C.c_void_p]
        L.rmi_delta_lower_bound.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_delta_upper_bound.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_delta_equal_range.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
        L.rmi_delta_range_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_delta_merge.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        _lib = L
    return _lib


def version() -> str:
    return load_library().rmi_version().decode()


def kernel_launch_count() -> int:
    return int(load_library().rmi_kernel_launch_count())


def _check(rc: int):
    if rc == 0:
        return
    msg = load_library().rmi_last_error().decode()
    if rc == 1:
        raise RMIPanic(msg)
    raise RMIError(f"rmi_b200 error {rc}: {msg}")


def _key_type_of(dtype) -> int:
    dtype = np.dtype(dtype)
    for kt, nd in _NP_OF_KEY.items():
        if dtype == np.dtype(nd):
            return kt
    raise TypeError(f"unsupported key dtype {dtype} (uint64, uint32, float64)")


class RMITrainingData:
    """A sorted key set resident in HBM (reference RMITrainingData, models/mod.rs:233-317).

    ``RMITrainingData(host_array)`` copies a numpy array to the device;
    ``RMITrainingData.from_device(ptr, n, key_type)`` borrows device memory (e.g. a torch
    tensor's ``data_ptr()``), no copy.
    """

    def __init__(self, keys: np.ndarray, device: int = 0):
        keys = np.ascontiguousarray(keys)
        self._h = C.c_void_p()
        self.key_type = _key_type_of(keys.dtype)
        self.device = int(device)
        self._keep = None
        _check(load_library().rmi_dataset_create(keys.ctypes.data_as(C.c_void_p), keys.size, self.key_type, device,
                                                 C.byref(self._h)))

    @classmethod
    def from_device(cls, ptr: int, n: int, key_type: int, device: int = 0, keep_alive=None) -> "RMITrainingData":
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self.key_type = key_type
        self.device = int(device)
        self._keep = keep_alive
        _check(load_library().rmi_dataset_wrap_device(C.c_void_p(ptr), n, key_type, device, C.byref(self._h)))
        return self

    @classmethod
    def from_file(cls, path: str, key_type: int = -1, device: int = 0) -> "RMITrainingData":
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self.device = int(device)
        self._keep = None
        _check(load_library().rmi_dataset_load_file(path.encode(), key_type, device, C.byref(self._h)))
        self.key_type = int(load_library().rmi_dataset_key_type(self._h))
        return self

    def replicate(self, device: int) -> "RMITrainingData":
        """A copy of this key set on another GPU (one device-to-device copy; RMITrainingData::soft_copy's
        role, models/mod.rs:311-316, for sweeps that spread independent builds over the GPUs of a node)."""
        other = type(self).__new__(type(self))
        other._h = C.c_void_p()
        other.key_type = self.key_type
        other.device = int(device)
        other._keep = None
        _check(load_library().rmi_dataset_replicate(self._h, int(device), C.byref(other._h)))
        return other

    def __len__(self) -> int:
        return int(load_library().rmi_dataset_len(self._h))

    def to_numpy(self) -> np.ndarray:
        """A host copy of the keys."""
        out = np.empty(len(self), dtype=_NP_OF_KEY[self.key_type])
        _check(load_library().rmi_dataset_copy_to_host(self._h, out.ctypes.data_as(C.c_void_p)))
        return out

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            load_library().rmi_dataset_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _take_knots(L, pts, cnt) -> np.ndarray:
    """Copy the library-owned knot array into a (K, 2) uint64 numpy array and release it."""
    try:
        n = int(cnt.value)
        return np.frombuffer((C.c_uint64 * (2 * n)).from_address(pts.value), dtype=np.uint64).reshape(n, 2).copy() if n \
            else np.zeros((0, 2), dtype=np.uint64)
    finally:
        L.rmi_spline_free(pts)


def cache_fix(data, line_size: int, with_stats: bool = False):
    """rmi_lib::cache_fix (cache_fix.rs:106-150): the error-bounded spline over key -> offset whose
    interpolation always lands in the key's line.  Returns the knots as a (K, 2) uint64 array of (key, offset).

    ``data`` is a numpy array (the reference's serial scan on one host core, no GPU) or an RMITrainingData (the
    same knots, fitted on the data's GPU from its resident keys).  with_stats=True returns ``(knots, stats)``:
    for the device scan a dict of rmi_cache_fix_stats (chunk_keys, chunks, points, stitch_segments,
    fallback_points, evaluations); None for the host scan."""
    L = load_library()
    pts, cnt = C.c_void_p(), C.c_uint64(0)
    if isinstance(data, RMITrainingData):
        st = _CacheFixStats()
        _check(L.rmi_cache_fix_device(data._h, int(line_size), C.byref(pts), C.byref(cnt), C.byref(st)))
        knots = _take_knots(L, pts, cnt)
        stats = {name: int(getattr(st, name)) for name, _ in _CacheFixStats._fields_}
        return (knots, stats) if with_stats else knots
    keys = np.ascontiguousarray(data)
    if keys.dtype != np.uint64:
        raise RMIPanic("Can only construct a bounded RMI on u64 data.")
    _check(L.rmi_cache_fix(keys.ctypes.data_as(C.c_void_p), keys.size, int(line_size), C.byref(pts), C.byref(cnt)))
    knots = _take_knots(L, pts, cnt)
    return (knots, None) if with_stats else knots


def train_bounded(data, model_spec: str, branch_factor: int, line_size: int, device: int = 0, flags: int = 0):
    """rmi_lib::train_bounded (train/mod.rs:156-184): cache_fix, then the two-layer RMI over the spline's knots
    on the GPU.  ``data``: a numpy array of uint64 keys (the cache-fix scan runs on the host) or an
    RMITrainingData (it runs on the data's GPU).  ``device`` is the GPU that trains the RMI over the knots.  Returns (TrainedRMI with
    num_data_rows = the number of keys, knots) — the pair the reference keeps in TrainedRMI.cache_fix."""
    knots = cache_fix(data, line_size)
    num_rows = len(data) if isinstance(data, RMITrainingData) else int(np.asarray(data).size)
    ds = RMITrainingData(np.ascontiguousarray(knots[:, 0]), device=device)
    try:
        rmi = train(ds, model_spec, branch_factor, flags)
    finally:
        ds.close()
    rmi.num_data_rows = num_rows
    return rmi, knots


def _result_ptr(rmi):
    """struct rmi_result* of a TrainedRMI returned by train() (or a ctypes _Result the caller filled in)."""
    if isinstance(rmi, _Result):
        return C.pointer(rmi)
    if rmi._res is None or rmi._res.res is None:
        raise RMIError("this TrainedRMI does not own a struct rmi_result")
    return rmi._res.res


def rmi_size(rmi, include_errors: bool = True, num_spline_points: int = 0) -> int:
    """rmi_lib::rmi_size (codegen.rs:375-394)."""
    return int(load_library().rmi_model_size(_result_ptr(rmi), int(include_errors), int(num_spline_points)))


def output_rmi(namespace: str, rmi, data_dir: str, key_type: int = KEY_U64, include_errors: bool = True, out_dir: str = ".",
               build_time_ns: int | None = None, cache_fix_knots: np.ndarray | None = None, line_size: int = 0,
               num_data_rows: int = 0) -> None:
    """rmi_lib::output_rmi (codegen.rs:757-788): <out_dir>/<ns>.cpp/.h/_data.h + <data_dir>/<ns>_L*_PARAMETERS.
    key_type is the KeyType handed to codegen (uint32 FILES keep KEY_U64, src/main.rs:122-132).
    cache_fix_knots: the (K, 2) array of a train_bounded() build."""
    os.makedirs(data_dir, exist_ok=True)
    ptr = _result_ptr(rmi)
    if build_time_ns is None:
        build_time_ns = int(ptr.contents.build_time_ns)
    knots = None if cache_fix_knots is None else np.ascontiguousarray(cache_fix_knots, dtype=np.uint64)
    _check(load_library().rmi_output_rmi(
        namespace.encode(), ptr, data_dir.encode(), out_dir.encode(), int(key_type), int(include_errors), int(build_time_ns),
        None if knots is None else knots.ctypes.data_as(C.c_void_p), 0 if knots is None else knots.shape[0], int(line_size),
        int(num_data_rows)))


def load_rmi(namespace: str, out_dir: str = ".", data_dir: str = "rmi_data"):
    """The inverse of output_rmi (host code, no GPU): reads <out_dir>/<ns>.cpp/.h/_data.h and the blobs under data_dir
    as the reference's code generator writes them.  Returns ``(TrainedRMI, cache_fix)``, cache_fix ``None`` or
    ``(line_size, knots)`` with knots a (K, 2) uint64 array (the reference's TrainedRMI.cache_fix).  The artefact holds
    no statistics (NaN / 0 here; ``evaluate`` measures them); ``last_layer_max_l1s`` is None for a --no-errors
    artefact.  linear, robust_linear and linear_spline generate the same code and load as linear.  ``key_type`` on
    the returned TrainedRMI is the lookup signature's (KEY_U64 or KEY_F64)."""
    L = load_library()
    res, pts, info = C.POINTER(_Result)(), C.c_void_p(), _ArtefactInfo()
    _check(L.rmi_load_rmi(namespace.encode(), out_dir.encode(), data_dir.encode(), C.byref(res), C.byref(pts), C.byref(info)))
    r = res.contents
    spec = f"{MODEL_NAMES[int(r.l0_model_id)]},{MODEL_NAMES[int(r.l1_model_id)]}"
    trained = result_from_pointer(res, spec)
    trained.num_data_rows = int(info.num_data_rows)
    trained.build_time = int(info.build_time_ns)
    trained.key_type = int(info.key_type)
    cf = None
    if pts.value:
        cf = (int(info.line_size), _take_knots(L, pts, C.c_uint64(info.num_knots)))
    return trained, cf


def evaluate(trained: TrainedRMI, data: RMITrainingData, counts: bool = True, flags: int = 0) -> TrainedRMI:
    """The reference's error pass, lower-bound widening and statistics (two_layer.rs:205-284) of ``trained``'s top and
    leaf tables over ``data``'s keys, on the GPU.  The tables are returned unchanged, bit for bit; the error bounds,
    the key counts (counts=True) and the statistics are those of ``data``, and num_rmi_rows = num_data_rows =
    len(data).  Raises RMIPanic where the top model is not monotone on ``data`` (two_layer.rs:50)."""
    if counts:
        flags = int(flags) | FLAG_LEAF_COUNTS
    res = C.POINTER(_Result)()
    _check(load_library().rmi_evaluate(data._h, _result_ptr(trained), int(flags), C.byref(res)))
    return result_from_pointer(res, trained.models)


def find_pareto_efficient_configs(replicas, restrict_to: int = 10, flags: int = 0) -> list[dict]:
    """optimizer::find_pareto_efficient_configs (optimizer.rs:233-249).  `replicas`: one RMITrainingData or a
    list holding the same keys on several devices (RMITrainingData.replicate); the independent stats-only
    builds are spread over them."""
    reps = [replicas] if isinstance(replicas, RMITrainingData) else list(replicas)
    handles = (C.c_void_p * len(reps))(*[r._h for r in reps])
    # The front can never hold more entries than configurations were measured (84 in phase 1 plus the
    # phase-2 refinements, optimizer.rs:110-231: a few hundred); 4096 is far above that, and a front that
    # still does not fit is an error, never a silent truncation (the dropped tail would be the smallest models).
    cap = max(4096, int(restrict_to) if restrict_to < (1 << 20) else 0)
    out = (_ConfigStats * cap)()
    cnt = C.c_uint64(0)
    _check(load_library().rmi_find_pareto_efficient_configs(handles, len(reps), int(restrict_to), int(flags), out, cap, C.byref(cnt)))
    if int(cnt.value) > cap:
        raise RMIError(f"Pareto front has {int(cnt.value)} entries, more than the {cap} this call can return")
    return [dict(models=out[i].models.decode(), branching_factor=int(out[i].branching_factor),
                 average_log2_error=float(out[i].average_log2_error), max_log2_error=float(out[i].max_log2_error),
                 size=int(out[i].size)) for i in range(int(cnt.value))]


def train_for_size(data: RMITrainingData, max_size: int, flags: int = 0) -> TrainedRMI:
    """rmi_lib::train_for_size (train/mod.rs:128-154): the first configuration of the (un-narrowed) Pareto
    front that is smaller than max_size bytes, trained in full."""
    front = find_pareto_efficient_configs(data, 1000, flags)
    pick = next((c for c in front if c["size"] < max_size), None)
    if pick is None:
        raise RMIPanic(f"Could not find any configurations smaller than {max_size}")
    return train(data, pick["models"], pick["branching_factor"], flags)


def load_data(path: str, key_type: int = -1, device: int = 0) -> RMITrainingData:
    """src/load.rs:132 load_data: header = u64 LE count, then packed keys; lands in HBM."""
    return RMITrainingData.from_file(path, key_type, device)


@dataclass
class TrainedRMI:
    """Owned copy of struct rmi_result; field names follow TrainedRMI (train/mod.rs:18-33)."""
    num_rmi_rows: int
    num_data_rows: int
    branching_factor: int
    model_avg_error: float
    model_avg_l2_error: float
    model_avg_log2_error: float
    model_max_log2_error: float
    model_max_error: int
    model_max_error_idx: int
    build_time: int               # ns, wall clock of the call
    device_time_ns: int
    phase_device_ns: tuple        # (top fit, leaf bounds, leaf fit+error pass, statistics)
    models: str
    l0_model: str
    l0_fparams: np.ndarray
    l0_iparams: np.ndarray
    l0_bradix_high: bool
    l0_table_bits: int
    l0_table32: np.ndarray | None
    l0_radix_index: np.ndarray | None
    l0_pivots: np.ndarray | None
    l1_model: str
    l1_params: np.ndarray | None   # (N, ppm)
    last_layer_max_l1s: np.ndarray | None
    l1_counts: np.ndarray | None
    could_not_replace: bool
    top_fit_exact: bool
    _res: object = None            # keeps the underlying struct rmi_result alive
    key_type: int | None = None    # load_rmi: the key type of the artefact's lookup signature


class _ResultOwner:
    """Owns a struct rmi_result*; freed (rmi_result_free) when the last array view is gone."""

    def __init__(self, res):
        self.res = res

    def __del__(self):
        try:
            if self.res is not None:
                load_library().rmi_result_free(self.res)
                self.res = None
        except Exception:
            pass


def _arr(ptr, n, ctype, dtype, owner):
    """Zero-copy numpy view of result memory owned by the library (keeps `owner` alive)."""
    n = int(n)
    if not ptr or n == 0:
        return None
    buf = (ctype * n).from_address(C.addressof(ptr.contents))
    buf._owner = owner
    return np.frombuffer(buf, dtype=dtype)


def train(data: RMITrainingData, model_spec: str, branch_factor: int, flags: int = 0,
          l0_params=None, counts: bool = True) -> TrainedRMI:
    """rmi_lib::train (train/mod.rs:100-126) on the GPU.  Raises RMIPanic where the reference panics.
    counts=True also fetches the per-leaf key counts (RMI_FLAG_LEAF_COUNTS, used by parity checks)."""
    L = load_library()
    if counts:
        flags = int(flags) | FLAG_LEAF_COUNTS
    res = C.POINTER(_Result)()
    if l0_params is None:
        rc = L.rmi_train(data._h, model_spec.encode(), int(branch_factor), int(flags), C.byref(res))
    else:
        p = np.ascontiguousarray(l0_params, dtype=np.float64)
        rc = L.rmi_train_with_top(data._h, model_spec.encode(), int(branch_factor), int(flags),
                                  p.ctypes.data_as(C.c_void_p), p.size, C.byref(res))
    _check(rc)
    return result_from_pointer(res, model_spec)


def train_stats_batch(data: RMITrainingData, top_model: str, leaf_models: list[str], branch_factor: int, flags: int = 0) -> list[TrainedRMI]:
    """rmi_train_stats_batch: the configurations "top,leaf_k" of one (top model, branching factor) in one call —
    one top-model fit and one boundary pass for all of them; statistics only (the optimizer's unit of work)."""
    L = load_library()
    L.rmi_train_stats_batch.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_char_p), C.c_int, C.c_uint64, C.c_uint32,
                                        C.POINTER(C.POINTER(_Result))]
    K = len(leaf_models)
    names = (C.c_char_p * K)(*[m.encode() for m in leaf_models])
    out = (C.POINTER(_Result) * K)()
    _check(L.rmi_train_stats_batch(data._h, top_model.encode(), names, K, int(branch_factor), int(flags), out))
    return [result_from_pointer(out[k], f"{top_model},{leaf_models[k]}") for k in range(K)]


def result_from_pointer(res, model_spec: str) -> TrainedRMI:
    """Wrap a struct rmi_result* returned by the library (zero-copy views, freed with the last view)."""
    if True:
        r = res.contents
        owner = _ResultOwner(res)
        N, ppm = int(r.branching_factor), int(r.l1_params_per_model)
        params = _arr(r.l1_params, N * ppm, C.c_double, np.float64, owner)
        out = TrainedRMI(
            num_rmi_rows=int(r.num_rmi_rows), num_data_rows=int(r.num_data_rows), branching_factor=N,
            model_avg_error=float(r.model_avg_error), model_avg_l2_error=float(r.model_avg_l2_error),
            model_avg_log2_error=float(r.model_avg_log2_error), model_max_log2_error=float(r.model_max_log2_error),
            model_max_error=int(r.model_max_error), model_max_error_idx=int(r.model_max_error_idx),
            build_time=int(r.build_time_ns), device_time_ns=int(r.device_time_ns),
            phase_device_ns=tuple(int(x) for x in r.phase_device_ns), models=model_spec,
            l0_model=MODEL_NAMES[int(r.l0_model_id)],
            l0_fparams=np.array(list(r.l0_fparams)[: int(r.l0_num_fparams)], dtype=np.float64),
            l0_iparams=np.array(list(r.l0_iparams)[: int(r.l0_num_iparams)], dtype=np.uint64),
            l0_bradix_high=bool(r.l0_bradix_high), l0_table_bits=int(r.l0_table_bits),
            l0_table32=_arr(r.l0_table32, r.l0_table32_len, C.c_uint32, np.uint32, owner),
            l0_radix_index=_arr(r.l0_array1, r.l0_array1_len, C.c_uint64, np.uint64, owner),
            l0_pivots=_arr(r.l0_array2, r.l0_array2_len, C.c_uint64, np.uint64, owner),
            l1_model=MODEL_NAMES[int(r.l1_model_id)],
            l1_params=None if params is None else params.reshape(N, ppm),
            last_layer_max_l1s=_arr(r.l1_errors, N, C.c_uint64, np.uint64, owner),
            l1_counts=_arr(r.l1_counts, N, C.c_uint64, np.uint64, owner),
            could_not_replace=bool(r.could_not_replace), top_fit_exact=bool(r.top_fit_exact), _res=owner)
    return out


class RMIIndex:
    """A trained RMI bound to the device-resident keys it was trained on, for batched lookups on the GPU.

    ``predict(q)`` returns the generated code's ``lookup(key, &err)`` for every query as ``(pos, err)``;
    ``lower_bound(q)`` returns the exact number of keys below each query (``std::lower_bound``), ``upper_bound(q)``
    the number of keys <= each query (``std::upper_bound``; 0 for NaN) and ``equal_range(q)`` both, from one window
    per query (DESIGN §18).  All take a numpy array of the dataset's key type and return ``np.uint64`` arrays.  The
    ``*_device`` forms take raw device
    pointers and a CUDA stream handle (torch: ``t.data_ptr()``, ``torch.cuda.current_stream().cuda_stream``) and
    enqueue one kernel without synchronising.  ``trained`` must hold its leaf tables (not FLAG_STATS_ONLY) and
    ``data`` must be the key set it was trained on; the index keeps ``data`` alive.
    """

    def __init__(self, trained: TrainedRMI, data: RMITrainingData):
        self._h = C.c_void_p()
        self.data = data
        self.key_type = data.key_type
        self._trained = trained
        _check(load_library().rmi_index_create(_result_ptr(trained), data._h, C.byref(self._h)))

    @classmethod
    def load(cls, namespace: str, data: RMITrainingData, out_dir: str = ".", data_dir: str = "rmi_data") -> "RMIIndex":
        """An index from generated artefacts (load_rmi) over ``data``: an RMIIndex, or a BoundedRMIIndex for a
        --bounded artefact.  An f64 artefact needs f64 data; a u64 artefact takes u64 or u32 data (the rmi CLI writes
        uint64_t code for uint32 key files).  A --no-errors artefact gets its bounds from ``evaluate`` on ``data``.
        Keys that differ in number from the ones the artefact was built on fail in rmi_index_create; an index over
        the new keys is then ``RMIIndex(evaluate(trained, data), data)``."""
        trained, cf = load_rmi(namespace, out_dir, data_dir)
        want = (KEY_F64,) if trained.key_type == KEY_F64 else (KEY_U64, KEY_U32)
        if data.key_type not in want:
            raise RMIError(f"the artefact's lookup takes {'double' if trained.key_type == KEY_F64 else 'uint64_t'} keys, "
                           f"the data holds {np.dtype(_NP_OF_KEY[data.key_type])}")
        if cf is not None:
            if trained.last_layer_max_l1s is None:
                raise RMIError("a --bounded artefact without errors cannot be served")
            return BoundedRMIIndex(trained, cf[1], cf[0], data)
        if trained.last_layer_max_l1s is None:
            trained = evaluate(trained, data, counts=False)
        return cls(trained, data)

    def _queries(self, q) -> np.ndarray:
        if not isinstance(q, np.ndarray) or q.dtype != np.dtype(_NP_OF_KEY[self.key_type]):
            got = q.dtype if isinstance(q, np.ndarray) else type(q).__name__
            raise TypeError(f"queries must be a numpy array of {np.dtype(_NP_OF_KEY[self.key_type])}, got {got}")
        return np.ascontiguousarray(q)

    def predict(self, q: np.ndarray):
        """(pos, err) per query, as np.uint64 arrays."""
        q = self._queries(q)
        pos = np.empty(q.size, dtype=np.uint64)
        err = np.empty(q.size, dtype=np.uint64)
        _check(load_library().rmi_index_lookup_host(self._h, q.ctypes.data_as(C.c_void_p), q.size, 0,
                                                     pos.ctypes.data_as(C.c_void_p), err.ctypes.data_as(C.c_void_p),
                                                     None))
        return pos, err

    def lower_bound(self, q: np.ndarray, return_fallbacks: bool = False):
        """Exact lower bound per query (np.uint64); with return_fallbacks also the number of queries whose
        error window missed the answer."""
        q = self._queries(q)
        out = np.empty(q.size, dtype=np.uint64)
        fb = C.c_uint64(0)
        _check(load_library().rmi_index_lookup_host(self._h, q.ctypes.data_as(C.c_void_p), q.size, 1,
                                                     out.ctypes.data_as(C.c_void_p), None, C.byref(fb)))
        return (out, int(fb.value)) if return_fallbacks else out

    def upper_bound(self, q: np.ndarray, return_fallbacks: bool = False):
        """Exact upper bound per query (np.uint64): the number of keys <= q, 0 for NaN; with return_fallbacks also
        the number of queries whose error window missed the answer."""
        q = self._queries(q)
        last = np.empty(q.size, dtype=np.uint64)
        fb = C.c_uint64(0)
        _check(load_library().rmi_index_range_host(self._h, q.ctypes.data_as(C.c_void_p), q.size, None,
                                                    last.ctypes.data_as(C.c_void_p), C.byref(fb)))
        return (last, int(fb.value)) if return_fallbacks else last

    def equal_range(self, q: np.ndarray, return_fallbacks: bool = False):
        """(first, last) per query, the half-open range of keys equal to q: first is lower_bound(q), last is
        upper_bound(q); with return_fallbacks also the number of queries whose window missed either end."""
        q = self._queries(q)
        first = np.empty(q.size, dtype=np.uint64)
        last = np.empty(q.size, dtype=np.uint64)
        fb = C.c_uint64(0)
        _check(load_library().rmi_index_range_host(self._h, q.ctypes.data_as(C.c_void_p), q.size,
                                                    first.ctypes.data_as(C.c_void_p), last.ctypes.data_as(C.c_void_p),
                                                    C.byref(fb)))
        return (first, last, int(fb.value)) if return_fallbacks else (first, last)

    def predict_device(self, q_ptr: int, n: int, pos_ptr: int, err_ptr: int = 0, stream: int = 0) -> None:
        _check(load_library().rmi_index_predict(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(pos_ptr),
                                                C.c_void_p(err_ptr or None), C.c_void_p(stream or None)))

    def lower_bound_device(self, q_ptr: int, n: int, out_ptr: int, fallbacks_ptr: int = 0, stream: int = 0) -> None:
        _check(load_library().rmi_index_lower_bound(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(out_ptr),
                                                    C.c_void_p(fallbacks_ptr or None), C.c_void_p(stream or None)))

    def upper_bound_device(self, q_ptr: int, n: int, out_ptr: int, fallbacks_ptr: int = 0, stream: int = 0) -> None:
        _check(load_library().rmi_index_upper_bound(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(out_ptr),
                                                    C.c_void_p(fallbacks_ptr or None), C.c_void_p(stream or None)))

    def equal_range_device(self, q_ptr: int, n: int, first_ptr: int, last_ptr: int, fallbacks_ptr: int = 0,
                           stream: int = 0) -> None:
        _check(load_library().rmi_index_equal_range(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(first_ptr),
                                                    C.c_void_p(last_ptr), C.c_void_p(fallbacks_ptr or None),
                                                    C.c_void_p(stream or None)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            load_library().rmi_index_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BoundedRMIIndex(RMIIndex):
    """A ``--bounded`` RMI bound to its keys: ``trained`` and ``knots`` are the pair ``train_bounded`` returns (the
    RMI over the cache-fix spline's knots and the ``(K, 2)`` uint64 knot array), ``data`` the uint64 keys the spline
    was fitted to.  ``predict`` returns the generated spline ``lookup(key, &err)`` (position rounded down to its
    line, ``err = line_size``); ``lower_bound`` is exact and, for a key of the data set, searches only that key's
    line.  Everything else is as for ``RMIIndex``; the knots are copied to the device."""

    def __init__(self, trained: TrainedRMI, knots: np.ndarray, line_size: int, data: RMITrainingData):
        self._h = C.c_void_p()
        self.data = data
        self.key_type = data.key_type
        self._trained = trained
        self.line_size = int(line_size)
        k = np.ascontiguousarray(knots, dtype=np.uint64)
        self.knots = k
        if k.ndim != 2 or k.shape[1] != 2:
            raise ValueError(f"knots must be a (K, 2) array of (key, offset), got shape {k.shape}")
        _check(load_library().rmi_index_create_bounded(_result_ptr(trained), k.ctypes.data_as(C.c_void_p), k.shape[0],
                                                       self.line_size, data._h, C.byref(self._h)))


class DeltaRMIIndex:
    """An updatable index (DESIGN §19): an ``RMIIndex`` or ``BoundedRMIIndex`` (kept alive here) and two sorted arrays
    on the index's device, the keys inserted since it was built and the keys removed since.  The logical key set is the
    multiset base ⊎ inserted ⊖ removed, and ``lower_bound``, ``upper_bound`` and ``equal_range`` are exact over it: the
    base index's answer plus the number of inserted keys below (or, for the upper bound, not above) the query, minus the
    number of removed keys below (not above) it.  Equal keys keep base keys first, then inserted keys in insert order,
    and a removal of a value takes away the first copy of its run, so ``merged_keys()`` is the stable sort of the base
    keys followed by every inserted batch, without the first c copies of each value removed c times.  There is no
    ``predict``: the model's positions refer to the base keys only.

    ``insert`` and ``remove`` must not run while another call on the same object, or a lookup it enqueued, is still in
    flight; lookups may run concurrently on several streams.  ``len(d)`` is n + m - t, ``num_inserted`` is m and
    ``num_removed`` is t."""

    def __init__(self, index: RMIIndex):
        self._h = C.c_void_p()
        self.index = index
        self.key_type = index.key_type
        _check(load_library().rmi_delta_create(index._h, C.byref(self._h)))

    @property
    def num_inserted(self) -> int:
        return int(load_library().rmi_delta_len(self._h))

    @property
    def num_removed(self) -> int:
        return int(load_library().rmi_delta_removed_len(self._h))

    def __len__(self) -> int:
        return len(self.index.data) + self.num_inserted - self.num_removed

    def insert(self, keys) -> None:
        """Merges a batch into the delta and returns when it is there.  ``keys``: a numpy array of the index's key type
        (sorted here with a stable sort, then copied to the device), or an RMITrainingData on the index's device (for
        device-resident batches, RMITrainingData.from_device), which must already be sorted.  A batch that is refused
        (unsorted, another key type or device, a NaN) leaves the delta unchanged."""
        self._apply(load_library().rmi_delta_insert, keys)

    def remove(self, keys) -> None:
        """Removes one copy of each key's value from the logical key set and returns when that is done.  ``keys`` as
        for ``insert``.  Refused with RMIError, changing nothing: a batch that is unsorted, of another key type or
        device, holds a NaN, or holds a value more often than the logical key set does (a key that is not there, one
        copy too many, a copy already removed)."""
        self._apply(load_library().rmi_delta_remove, keys)

    def _apply(self, call, keys):
        if isinstance(keys, RMITrainingData):
            _check(call(self._h, keys._h))
            return
        if not isinstance(keys, np.ndarray) or keys.dtype != np.dtype(_NP_OF_KEY[self.key_type]):
            got = keys.dtype if isinstance(keys, np.ndarray) else type(keys).__name__
            raise TypeError(f"keys must be a numpy array of {np.dtype(_NP_OF_KEY[self.key_type])}, got {got}")
        batch = RMITrainingData(np.sort(keys.ravel(), kind="stable"),
                                device=self.index.data.device)
        try:
            _check(call(self._h, batch._h))
        finally:
            batch.close()

    def lower_bound(self, q: np.ndarray, return_fallbacks: bool = False):
        """Exact lower bound over the logical key set per query (np.uint64); with return_fallbacks also the base
        index's fallback count."""
        first, _, fb = self._range(q, True, False)
        return (first, fb) if return_fallbacks else first

    def upper_bound(self, q: np.ndarray, return_fallbacks: bool = False):
        """Exact upper bound over the logical key set per query (np.uint64), 0 for NaN."""
        _, last, fb = self._range(q, False, True)
        return (last, fb) if return_fallbacks else last

    def equal_range(self, q: np.ndarray, return_fallbacks: bool = False):
        """(first, last) per query over the logical key set."""
        first, last, fb = self._range(q, True, True)
        return (first, last, fb) if return_fallbacks else (first, last)

    def _range(self, q, want_first, want_last):
        q = self.index._queries(q)
        first = np.empty(q.size, dtype=np.uint64) if want_first else None
        last = np.empty(q.size, dtype=np.uint64) if want_last else None
        fb = C.c_uint64(0)
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        _check(load_library().rmi_delta_range_host(self._h, q.ctypes.data_as(C.c_void_p), q.size, ptr(first), ptr(last),
                                                    C.byref(fb)))
        return first, last, int(fb.value)

    def lower_bound_device(self, q_ptr: int, n: int, out_ptr: int, fallbacks_ptr: int = 0, stream: int = 0) -> None:
        _check(load_library().rmi_delta_lower_bound(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(out_ptr),
                                                    C.c_void_p(fallbacks_ptr or None), C.c_void_p(stream or None)))

    def upper_bound_device(self, q_ptr: int, n: int, out_ptr: int, fallbacks_ptr: int = 0, stream: int = 0) -> None:
        _check(load_library().rmi_delta_upper_bound(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(out_ptr),
                                                    C.c_void_p(fallbacks_ptr or None), C.c_void_p(stream or None)))

    def equal_range_device(self, q_ptr: int, n: int, first_ptr: int, last_ptr: int, fallbacks_ptr: int = 0,
                           stream: int = 0) -> None:
        _check(load_library().rmi_delta_equal_range(self._h, C.c_void_p(q_ptr), int(n), C.c_void_p(first_ptr),
                                                    C.c_void_p(last_ptr), C.c_void_p(fallbacks_ptr or None),
                                                    C.c_void_p(stream or None)))

    def merged_keys(self) -> RMITrainingData:
        """The n + m - t logical keys, in the order the class describes, as a new RMITrainingData that owns them, on
        the index's device (its sortedness found by the same check as any data set's).  Empty when every key was
        removed."""
        out = RMITrainingData.__new__(RMITrainingData)
        out._h = C.c_void_p()
        out.key_type = self.key_type
        out.device = self.index.data.device
        out._keep = None
        _check(load_library().rmi_delta_merge(self._h, C.byref(out._h)))
        return out

    def compact(self, mode: str = "retrain") -> "DeltaRMIIndex":
        """A new DeltaRMIIndex with an empty delta over a fresh index on merged_keys(); this one stays valid until it is
        closed.  mode "retrain" trains the base's spec and branching factor again (train_bounded, with the cache-fix
        scan on the device, for a bounded base); "evaluate" keeps a plain base's tables and re-derives their error
        bounds on the merged keys (RMIPanic where the top model is not monotone on them).  A bounded base has no
        "evaluate": its knots belong to the old keys."""
        if mode not in ("retrain", "evaluate"):
            raise ValueError(f'mode must be "retrain" or "evaluate", got {mode!r}')
        base = self.index
        bounded = isinstance(base, BoundedRMIIndex)
        if bounded and mode == "evaluate":
            raise RMIError("a bounded index cannot be compacted by evaluation: its spline knots belong to the old keys")
        merged = self.merged_keys()
        t = base._trained
        if bounded:
            r, knots = train_bounded(merged, t.models, t.branching_factor, base.line_size, device=merged.device)
            return DeltaRMIIndex(BoundedRMIIndex(r, knots, base.line_size, merged))
        g = train(merged, t.models, t.branching_factor) if mode == "retrain" else evaluate(t, merged, counts=False)
        return DeltaRMIIndex(RMIIndex(g, merged))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            load_library().rmi_delta_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
