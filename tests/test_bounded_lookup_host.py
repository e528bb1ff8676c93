"""rmi_index_create_bounded refuses missing arguments on the host, before any device work (runs without a GPU)."""
import ctypes as C

import numpy as np


def test_index_create_bounded_rejects_null_arguments_without_a_device():
    import rmi_b200
    from rmi_b200.api import _Result
    L = rmi_b200.load_library()
    out = C.c_void_p()
    r = _Result()
    knots = np.zeros((4, 2), dtype=np.uint64)
    kp = knots.ctypes.data_as(C.c_void_p)
    fake_ds = C.c_void_p(1)                                            # never dereferenced: refused first
    for args in ((None, kp, 4, 8, fake_ds, C.byref(out)), (C.byref(r), None, 4, 8, fake_ds, C.byref(out)),
                 (C.byref(r), kp, 4, 8, None, C.byref(out)), (C.byref(r), kp, 4, 8, fake_ds, None)):
        assert L.rmi_index_create_bounded(*args) == 2                 # RMI_ERR_INVALID
        assert b"rmi_index_create_bounded: null" in L.rmi_last_error()
    assert not out.value
