"""Host-side checks of the upper-bound and equal-range calls (rmi_index_upper_bound, rmi_index_equal_range,
rmi_index_range_host): arguments are refused before any device work."""
import ctypes as C


def test_range_calls_refuse_bad_arguments_without_a_device():
    import rmi_b200
    L = rmi_b200.load_library()
    q = (C.c_uint64 * 4)()
    out = (C.c_uint64 * 4)()
    fb = C.c_uint64(7)
    assert L.rmi_index_upper_bound(None, q, 4, out, None, None) == 2                  # RMI_ERR_INVALID
    assert b"rmi_index_upper_bound: null index" in L.rmi_last_error()
    assert L.rmi_index_equal_range(None, q, 4, out, out, None, None) == 2
    assert b"rmi_index_equal_range: null index" in L.rmi_last_error()
    assert L.rmi_index_range_host(None, q, 4, None, out, C.byref(fb)) == 2
    assert b"rmi_index_range_host: null index" in L.rmi_last_error()
    fake = C.c_void_p(1)                                                               # never dereferenced
    assert L.rmi_index_upper_bound(fake, q, 4, None, None, None) == 2
    assert b"null query or output pointer" in L.rmi_last_error()
    assert L.rmi_index_equal_range(fake, q, 4, None, out, None, None) == 2
    assert L.rmi_index_equal_range(fake, q, 4, out, None, None, None) == 2
    assert L.rmi_index_range_host(fake, None, 4, None, out, None) == 2
    # n == 0 needs no pointers and does no device work
    assert L.rmi_index_upper_bound(fake, None, 0, None, None, None) == 0
    assert L.rmi_index_equal_range(fake, None, 0, None, None, None, None) == 0
    assert L.rmi_index_range_host(fake, None, 0, None, None, C.byref(fb)) == 0
    assert fb.value == 0
