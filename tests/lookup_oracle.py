"""The CPU oracle's lookup on given tables (tests/cxx/oracle_tables.cpp): ``from_result(trained)`` rebuilds an
oracle RMI from the top model and leaf tables of a TrainedRMI (GPU) or an oracle.OracleRMI, so that its
``lookup_batch`` evaluates exactly those tables.  Test infrastructure, built into a directory the caller gives."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cxx", "oracle_tables.cpp")

_lib = None


def build(out_dir: str):
    """Compile the table oracle into out_dir with the oracle's flags and load it."""
    global _lib
    if _lib is None:
        so = os.path.join(out_dir, "liboracle_tables.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-pthread", "-shared", SRC, "-o", so],
                       check=True)
        L = C.CDLL(so)
        L.rmi_oracle_from_tables.restype = C.c_void_p
        L.rmi_oracle_from_tables.argtypes = ([C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
                                             + [C.c_void_p, C.c_uint64] * 3
                                             + [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_uint64])
        L.rmi_oracle_last_error.restype = C.c_char_p
        L.rmi_oracle_free.argtypes = [C.c_void_p]
        L.rmi_oracle_lookup_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _ptr(a):
    return None if a is None or a.size == 0 else a.ctypes.data_as(C.c_void_p)


def _arr(a, dtype):
    return np.zeros(0, dtype=dtype) if a is None else np.ascontiguousarray(a, dtype=dtype)


class TableRMI:
    def __init__(self, h):
        self._h = h

    def lookup_batch(self, keys: np.ndarray):
        keys = np.ascontiguousarray(keys)
        pos = np.zeros(keys.size, dtype=np.uint64)
        err = np.zeros(keys.size, dtype=np.uint64)
        _lib.rmi_oracle_lookup_batch(self._h, _ptr(keys), keys.size, oracle.key_type_of(keys), _ptr(pos), _ptr(err))
        return pos, err

    def close(self):
        if self._h:
            _lib.rmi_oracle_free(self._h)
            self._h = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def from_tables(top_kind: str, high: bool, table_bits: int, fp, ip, t32, a1, a2, leaf_kind: str, params, errors,
                n: int) -> TableRMI:
    assert _lib is not None, "call build() first"
    fp, ip = _arr(fp, np.float64), _arr(ip, np.uint64)
    t32, a1, a2 = _arr(t32, np.uint32), _arr(a1, np.uint64), _arr(a2, np.uint64)
    params, errors = np.ascontiguousarray(params, dtype=np.float64), np.ascontiguousarray(errors, dtype=np.uint64)
    N = errors.size
    ppm = params.size // N
    kinds = oracle.KINDS
    h = _lib.rmi_oracle_from_tables(kinds.index(top_kind), int(high), int(table_bits), _ptr(fp), fp.size, _ptr(ip),
                                    ip.size, _ptr(t32), t32.size, _ptr(a1), a1.size, _ptr(a2), a2.size,
                                    kinds.index(leaf_kind), _ptr(params), ppm, _ptr(errors), N, int(n))
    if not h:
        raise ValueError(_lib.rmi_oracle_last_error().decode())
    return TableRMI(h)


def from_result(trained) -> TableRMI:
    """An oracle RMI over the tables of `trained`: a GPU TrainedRMI or an oracle.OracleRMI."""
    if isinstance(trained, oracle.OracleRMI):
        l0 = trained.l0
        bits = int(np.log2(l0.t32.size)) if l0.kind == "radix_table" else 0
        return from_tables(l0.kind, l0.high, bits, l0.fp, l0.ip, l0.t32, l0.a1, l0.a2, trained.l1_kind,
                           trained.l1_params, trained.l1_errors, trained.n)
    return from_tables(trained.l0_model, trained.l0_bradix_high, trained.l0_table_bits, trained.l0_fparams,
                       trained.l0_iparams, trained.l0_table32, trained.l0_radix_index, trained.l0_pivots,
                       trained.l1_model, trained.l1_params, trained.last_layer_max_l1s, trained.num_rmi_rows)
