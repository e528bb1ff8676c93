"""rmi_cache_fix_device refuses null arguments on the host, before any device work (runs without a GPU)."""
import ctypes as C


def test_cache_fix_device_rejects_null_arguments_without_a_device():
    import rmi_b200
    L = rmi_b200.load_library()
    pts, cnt = C.c_void_p(), C.c_uint64(0)
    fake_ds = C.c_void_p(1)                                            # never dereferenced: refused first
    for args in ((None, 8, C.byref(pts), C.byref(cnt), None), (fake_ds, 8, None, C.byref(cnt), None),
                 (fake_ds, 8, C.byref(pts), None, None)):
        assert L.rmi_cache_fix_device(*args) == 2                     # RMI_ERR_INVALID
        assert b"rmi_cache_fix_device: null argument" in L.rmi_last_error()
    assert not pts.value and cnt.value == 0
