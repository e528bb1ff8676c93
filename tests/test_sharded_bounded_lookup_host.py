"""rmi_shard_index_create_bounded and the collective predict calls refuse missing arguments on the host, before any
device work (runs without a GPU)."""
import ctypes as C

import numpy as np


def test_shard_index_create_bounded_rejects_null_arguments_without_a_device():
    import rmi_b200
    from rmi_b200.api import _Result
    L = rmi_b200.load_library()
    L.rmi_shard_index_create_bounded.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p,
                                                 C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    out = C.c_void_p()
    r = _Result()
    knots = np.zeros((4, 2), dtype=np.uint64)
    counts = np.array([4], dtype=np.uint64)
    ends = np.zeros(5, dtype=np.uint64)
    kp, cp, ep = (a.ctypes.data_as(C.c_void_p) for a in (knots, counts, ends))
    fake_ds = C.c_void_p(1)                                            # never dereferenced: refused first
    full = [C.byref(r), kp, 4, 0, cp, 8, fake_ds, ep, 1, 0, C.byref(out)]
    for k in (0, 1, 4, 6, 7, 10):                                      # result, knots, counts, local, ends, out
        args = list(full)
        args[k] = None
        assert L.rmi_shard_index_create_bounded(*args) == 2           # RMI_ERR_INVALID
        assert b"rmi_shard_index_create_bounded: null argument" in L.rmi_last_error()
    assert not out.value


def test_shard_index_predict_calls_reject_a_null_index_without_a_device():
    import rmi_b200
    L = rmi_b200.load_library()
    q = C.c_void_p(1)
    L.rmi_shard_index_predict_route.argtypes = [C.c_void_p] * 2 + [C.c_uint64] + [C.c_void_p] * 4
    L.rmi_shard_index_predict_search.argtypes = [C.c_void_p] * 2 + [C.c_uint64] + [C.c_void_p] * 2
    L.rmi_shard_index_predict_collective.argtypes = [C.c_void_p] * 3 + [C.c_uint64] + [C.c_void_p] * 3
    calls = (("rmi_shard_index_predict_route", (None, q, 1, q, q, q, None)),
             ("rmi_shard_index_predict_search", (None, q, 1, q, None)),
             ("rmi_shard_index_predict_collective", (None, q, q, 1, q, None, None)))
    for name, args in calls:
        assert getattr(L, name)(*args) == 2
        assert L.rmi_last_error().decode() == f"{name}: null index"
