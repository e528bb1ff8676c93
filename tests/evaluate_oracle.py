"""The CPU oracle's error pass over given tables (tests/cxx/oracle_evaluate.cpp): ``evaluate(trained, keys)`` returns
the errors, counts and statistics the reference's two_layer.rs:178-284 computes for ``trained``'s tables on ``keys``,
without the empty-leaf constant replacement.  Test infrastructure, built into a directory the caller gives."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cxx", "oracle_evaluate.cpp")

_lib = None


def build(out_dir: str):
    """Compile the evaluate oracle into out_dir with the oracle's flags and load it."""
    global _lib
    if _lib is None:
        so = os.path.join(out_dir, "liboracle_evaluate.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-pthread", "-shared", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        # the table oracle's constructor is part of the same library (oracle_evaluate.cpp includes oracle_tables.cpp)
        L.rmi_oracle_from_tables.restype = C.c_void_p
        L.rmi_oracle_from_tables.argtypes = ([C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
                                             + [C.c_void_p, C.c_uint64] * 3
                                             + [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_uint64])
        L.rmi_oracle_evaluate.restype = C.c_void_p
        L.rmi_oracle_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int]
        L.rmi_oracle_last_error.restype = C.c_char_p
        L.rmi_oracle_free.argtypes = [C.c_void_p]
        L.rmi_oracle_summary.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_oracle_l1_get.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        _lib = L
    return _lib


@dataclass
class Evaluated:
    errors: np.ndarray
    counts: np.ndarray
    max_error: int
    max_error_idx: int
    avg_error: float
    avg_l2_error: float
    avg_log2_error: float
    max_log2_error: float


def _p(a):
    return None if a is None or a.size == 0 else a.ctypes.data_as(C.c_void_p)


def _arr(a, dtype):
    return np.zeros(0, dtype=dtype) if a is None else np.ascontiguousarray(a, dtype=dtype)


def evaluate(trained, keys: np.ndarray) -> Evaluated:
    """Raises oracle.OraclePanic where the reference panics (a top model that is not monotone on the keys)."""
    assert _lib is not None, "call build() first"
    if isinstance(trained, oracle.OracleRMI):
        l0 = trained.l0
        t = (l0.kind, l0.high, int(np.log2(l0.t32.size)) if l0.kind == "radix_table" else 0, l0.fp, l0.ip, l0.t32, l0.a1,
             l0.a2, trained.l1_kind, trained.l1_params, trained.n)
    else:
        t = (trained.l0_model, trained.l0_bradix_high, trained.l0_table_bits, trained.l0_fparams, trained.l0_iparams,
             trained.l0_table32, trained.l0_radix_index, trained.l0_pivots, trained.l1_model, trained.l1_params,
             trained.num_rmi_rows)
    top, high, bits, fp, ip, t32, a1, a2, leaf, params, n = t
    fp, ip, t32, a1, a2 = _arr(fp, np.float64), _arr(ip, np.uint64), _arr(t32, np.uint32), _arr(a1, np.uint64), _arr(a2, np.uint64)
    params = np.ascontiguousarray(params, dtype=np.float64)
    N = params.shape[0]
    errors = np.zeros(N, dtype=np.uint64)   # the given bounds play no part in the pass
    kinds = oracle.KINDS
    h = _lib.rmi_oracle_from_tables(kinds.index(top), int(high), int(bits), _p(fp), fp.size, _p(ip), ip.size, _p(t32),
                                    t32.size, _p(a1), a1.size, _p(a2), a2.size, kinds.index(leaf), _p(params),
                                    params.shape[1], _p(errors), N, int(n))
    if not h:
        raise ValueError(_lib.rmi_oracle_last_error().decode())
    try:
        keys = np.ascontiguousarray(keys)
        e = _lib.rmi_oracle_evaluate(h, _p(keys), keys.size, oracle.key_type_of(keys))
        if not e:
            raise oracle.OraclePanic(_lib.rmi_oracle_last_error().decode())
    finally:
        _lib.rmi_oracle_free(h)
    try:
        scal = np.zeros(8, dtype=np.uint64)
        stats = np.zeros(4, dtype=np.float64)
        _lib.rmi_oracle_summary(e, _p(scal), _p(stats))
        out_e, out_c = np.zeros(N, dtype=np.uint64), np.zeros(N, dtype=np.uint64)
        _lib.rmi_oracle_l1_get(e, None, _p(out_e), _p(out_c))
    finally:
        _lib.rmi_oracle_free(e)
    return Evaluated(out_e, out_c, int(scal[2]), int(scal[3]), float(stats[0]), float(stats[1]), float(stats[2]),
                     float(stats[3]))
