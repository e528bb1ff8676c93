"""ctypes binding for the CPU oracle (oracle/librmi_oracle.so).

TEST INFRASTRUCTURE ONLY.  Importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; the product package rmi_b200 never imports it.
See the header of oracle/rmi_oracle.cpp for what the oracle restates and how it is pinned.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "librmi_oracle.so")

KEY_U64, KEY_U32, KEY_F64 = 0, 1, 2
_KEY_DTYPES = {KEY_U64: np.uint64, KEY_U32: np.uint32, KEY_F64: np.float64}

KINDS = ["linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal",
         "radix", "radix_table", "bradix", "histogram"]


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (g++, seconds)."""
    src = os.path.join(_HERE, "rmi_oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE], check=True, stdout=subprocess.DEVNULL)
    return _LIB_PATH


def build_variant(out_dir: str, *defines: str):
    """A test-only variant of the oracle, compiled into out_dir with the given -D macros (e.g. ORACLE_FIT_LN_NOISE)
    and loaded: pass it to train(..., library=...)."""
    so = os.path.join(os.path.abspath(out_dir), "librmi_oracle.so")
    subprocess.run(["make", "-C", _HERE, f"OUT={so}", "DEFINES=" + " ".join(f"-D{d}" for d in defines)], check=True,
                   stdout=subprocess.DEVNULL)
    return _bind(C.CDLL(so))


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = _bind(C.CDLL(_LIB_PATH))
    return _lib


def _bind(L):
    L.rmi_oracle_train.restype = C.c_void_p
    L.rmi_oracle_train.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_char_p, C.c_uint64,
                                   C.c_void_p, C.c_int, C.c_int]
    L.rmi_oracle_last_error.restype = C.c_char_p
    L.rmi_oracle_free.argtypes = [C.c_void_p]
    L.rmi_oracle_summary.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.rmi_oracle_l0_sizes.argtypes = [C.c_void_p, C.c_void_p]
    L.rmi_oracle_l0_get.argtypes = [C.c_void_p] + [C.c_void_p] * 5
    L.rmi_oracle_l1_params_per_model.restype = C.c_uint32
    L.rmi_oracle_l1_params_per_model.argtypes = [C.c_void_p]
    L.rmi_oracle_l1_get.argtypes = [C.c_void_p] + [C.c_void_p] * 3
    L.rmi_oracle_lookup.restype = C.c_uint64
    L.rmi_oracle_lookup.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_double, C.c_void_p]
    L.rmi_oracle_lookup_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
    L.rmi_oracle_model_train.restype = C.c_void_p
    L.rmi_oracle_model_train.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_double]
    L.rmi_oracle_model_free.argtypes = [C.c_void_p]
    L.rmi_oracle_model_predict_int.restype = C.c_uint64
    L.rmi_oracle_model_predict_int.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_double]
    L.rmi_oracle_model_predict_float.restype = C.c_double
    L.rmi_oracle_model_predict_float.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_double]
    L.rmi_oracle_model_sizes.argtypes = [C.c_void_p, C.c_void_p]
    L.rmi_oracle_model_get.argtypes = [C.c_void_p] + [C.c_void_p] * 5
    L.rmi_oracle_model_high.restype = C.c_int
    L.rmi_oracle_model_high.argtypes = [C.c_void_p]
    L.rmi_oracle_scale_offset.restype = C.c_uint64
    L.rmi_oracle_scale_offset.argtypes = [C.c_uint64, C.c_double]
    L.rmi_oracle_set_trailing_repeat.argtypes = [C.c_int]
    L.rmi_oracle_common_prefix_u64.restype = C.c_uint8
    L.rmi_oracle_common_prefix_u64.argtypes = [C.c_void_p, C.c_uint64]
    return L


class OraclePanic(RuntimeError):
    """The reference would have panicked on this input."""


def key_type_of(keys: np.ndarray) -> int:
    if keys.dtype == np.uint64:
        return KEY_U64
    if keys.dtype == np.uint32:
        return KEY_U32
    if keys.dtype == np.float64:
        return KEY_F64
    raise TypeError(f"unsupported key dtype {keys.dtype}")


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@dataclass
class ModelParams:
    kind: str
    fp: np.ndarray
    ip: np.ndarray
    t32: np.ndarray
    a1: np.ndarray
    a2: np.ndarray
    high: bool = True


@dataclass
class OracleRMI:
    """Mirror of TrainedRMI (train/mod.rs:18-33) as produced by the oracle."""
    n: int
    branching_factor: int
    max_error: int
    max_error_idx: int
    avg_error: float
    avg_l2_error: float
    avg_log2_error: float
    max_log2_error: float
    l0: ModelParams
    l1_kind: str
    l1_params: np.ndarray        # (N, ppm) float64
    l1_errors: np.ndarray        # (N,) uint64
    l1_counts: np.ndarray        # (N,) uint64
    could_not_replace: bool = False
    _handle: int = field(default=0, repr=False)
    _lib: object = field(default=None, repr=False)   # the library that made it (a build_variant one, or None)

    def lookup(self, key) -> tuple[int, int]:
        err = C.c_uint64(0)
        isf = isinstance(key, float)
        pos = (self._lib or lib()).rmi_oracle_lookup(self._handle, int(isf), 0 if isf else int(key), float(key) if isf else 0.0,
                                      C.byref(err))
        return int(pos), int(err.value)

    def lookup_batch(self, keys: np.ndarray):
        keys = np.ascontiguousarray(keys)
        pos = np.zeros(keys.size, dtype=np.uint64)
        err = np.zeros(keys.size, dtype=np.uint64)
        (self._lib or lib()).rmi_oracle_lookup_batch(self._handle, _ptr(keys), keys.size, key_type_of(keys), _ptr(pos), _ptr(err))
        return pos, err

    def close(self):
        if self._handle:
            (self._lib or lib()).rmi_oracle_free(self._handle)
            self._handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _get_model(sizes_fn, get_fn, h, kind, high=True) -> ModelParams:
    sizes = np.zeros(5, dtype=np.uint64)
    sizes_fn(h, _ptr(sizes))
    fp = np.zeros(int(sizes[0]), dtype=np.float64)
    ip = np.zeros(int(sizes[1]), dtype=np.uint64)
    t32 = np.zeros(int(sizes[2]), dtype=np.uint32)
    a1 = np.zeros(int(sizes[3]), dtype=np.uint64)
    a2 = np.zeros(int(sizes[4]), dtype=np.uint64)
    get_fn(h, _ptr(fp), _ptr(ip), _ptr(t32), _ptr(a1), _ptr(a2))
    return ModelParams(kind, fp, ip, t32, a1, a2, high)


def train(keys: np.ndarray, model_spec: str, branch_factor: int, l0_override=None, threads: int = 2,
          library=None) -> OracleRMI:
    """rmi_lib::train (train/mod.rs:100) on an in-memory sorted key array (with `library` from build_variant: the
    variant's train)."""
    keys = np.ascontiguousarray(keys)
    kt = key_type_of(keys)
    L = library or lib()
    ov = None if l0_override is None else np.ascontiguousarray(l0_override, dtype=np.float64)
    h = L.rmi_oracle_train(_ptr(keys), keys.size, kt, model_spec.encode(), int(branch_factor),
                           _ptr(ov), 0 if ov is None else ov.size, threads)
    if not h:
        raise OraclePanic(L.rmi_oracle_last_error().decode())
    scal = np.zeros(8, dtype=np.uint64)
    stats = np.zeros(4, dtype=np.float64)
    L.rmi_oracle_summary(h, _ptr(scal), _ptr(stats))
    N = int(scal[1])
    ppm = int(L.rmi_oracle_l1_params_per_model(h))
    params = np.zeros((N, ppm), dtype=np.float64)
    errors = np.zeros(N, dtype=np.uint64)
    counts = np.zeros(N, dtype=np.uint64)
    L.rmi_oracle_l1_get(h, _ptr(params), _ptr(errors), _ptr(counts))
    l0 = _get_model(L.rmi_oracle_l0_sizes, L.rmi_oracle_l0_get, h, KINDS[int(scal[4])], bool(scal[6]))
    return OracleRMI(n=int(scal[0]), branching_factor=N, max_error=int(scal[2]), max_error_idx=int(scal[3]),
                     avg_error=float(stats[0]), avg_l2_error=float(stats[1]), avg_log2_error=float(stats[2]),
                     max_log2_error=float(stats[3]), l0=l0, l1_kind=KINDS[int(scal[5])], l1_params=params,
                     l1_errors=errors, l1_counts=counts, could_not_replace=bool(scal[7]), _handle=h, _lib=library)


class OracleModel:
    """One model trained by train_model (train/mod.rs:35-57) on explicit (key, offset) pairs."""

    def __init__(self, name: str, keys, offsets=None, scale: float = 1.0, dtype=np.uint64):
        keys = np.ascontiguousarray(keys, dtype=dtype)
        offs = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.uint64)
        self._is_float = keys.dtype == np.float64
        L = lib()
        self._h = L.rmi_oracle_model_train(name.encode(), _ptr(keys), _ptr(offs), keys.size, key_type_of(keys),
                                           float(scale))
        if not self._h:
            raise OraclePanic(L.rmi_oracle_last_error().decode())
        self.params = _get_model(L.rmi_oracle_model_sizes, L.rmi_oracle_model_get, self._h, name,
                                 bool(L.rmi_oracle_model_high(self._h)))

    def predict_to_int(self, key) -> int:
        if self._is_float:
            return int(lib().rmi_oracle_model_predict_int(self._h, 1, 0, float(key)))
        return int(lib().rmi_oracle_model_predict_int(self._h, 0, int(key), 0.0))

    def predict_to_float(self, key) -> float:
        if self._is_float:
            return float(lib().rmi_oracle_model_predict_float(self._h, 1, 0, float(key)))
        return float(lib().rmi_oracle_model_predict_float(self._h, 0, int(key), 0.0))

    def __del__(self):
        try:
            if self._h:
                lib().rmi_oracle_model_free(self._h)
                self._h = 0
        except Exception:
            pass


def scale_offset(off: int, scale: float) -> int:
    return int(lib().rmi_oracle_scale_offset(int(off), float(scale)))


def set_trailing_repeat(on: bool) -> None:
    """Test knob: switch off FixDupsIter's trailing repeated item (models/mod.rs:180)."""
    lib().rmi_oracle_set_trailing_repeat(int(bool(on)))


def common_prefix_u64(keys) -> int:
    k = np.ascontiguousarray(keys, dtype=np.uint64)
    return int(lib().rmi_oracle_common_prefix_u64(_ptr(k), k.size))
