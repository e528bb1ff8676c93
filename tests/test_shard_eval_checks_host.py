"""rmi_shard_eval_create runs the shared check of a given result (tests/test_result_checks_host.py) and the ends-table
checks of rmi_shard_index_create before any device work, and rmi_shard_build_create makes the same ends-table checks:
each refusal gives its code and message with a zero-filled host block as the dataset, which a check that touched the
device or the keys would not survive."""
import ctypes as C

import pytest

from tests.test_result_checks_host import DEFECTS, INVALID, LINEAR, SHARED_TEXTS, _result

FN = "rmi_shard_eval_create"
PANIC = 1


@pytest.fixture(scope="module")
def lib():
    import rmi_b200
    L = rmi_b200.load_library()
    from rmi_b200 import sharded
    L.rmi_shard_eval_create.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(sharded._Ends), C.c_int, C.c_int,
                                        C.POINTER(C.c_void_p)]
    L.rmi_shard_build_create.argtypes = [C.c_void_p, C.POINTER(sharded._Ends), C.c_int, C.c_int, C.c_char_p, C.c_uint64,
                                         C.c_uint64, C.POINTER(sharded._Buffers), C.c_void_p, C.POINTER(C.c_void_p)]
    return L


def _dataset(n=0, sorted_=1):
    """A host block laid out as rmi_dataset (d_keys, n, key_type, device, owned, pooled, sorted, no_dups)."""
    block = (C.c_uint64 * 8)()
    block[1] = n
    C.memmove(C.addressof(block) + 26, bytes([sorted_]), 1)
    return block


def _ends(*rows):
    from rmi_b200 import sharded
    return (sharded._Ends * len(rows))(*[sharded._Ends(*r) for r in rows])


def _create(L, r, block, ends, world, rank):
    h = C.c_void_p()
    rc = L.rmi_shard_eval_create(C.byref(r), C.c_void_p(C.addressof(block)), ends, world, rank, C.byref(h))
    assert rc != 0, "refusals only: a created evaluator would have done device work"
    return rc, L.rmi_last_error().decode()


def _create_build(L, block, ends, world, rank):
    from rmi_b200 import sharded
    h = C.c_void_p()
    rc = L.rmi_shard_build_create(C.c_void_p(C.addressof(block)), ends, world, rank, b"linear,linear", 64, 0,
                                  C.byref(sharded._Buffers()), None, C.byref(h))
    assert rc != 0, "refusals only: a created build would have done device work"
    return rc, L.rmi_last_error().decode()


# the evaluation re-derives the error bounds, so (as for rmi_evaluate) a result without them is accepted
CASES = [pytest.param(*d[1:6], id=d[0]) for d in DEFECTS if not d[6]]


@pytest.mark.parametrize("top,bits,defect,code,text", CASES)
def test_refuses_a_malformed_result_like_the_other_consumers(lib, top, bits, defect, code, text):
    r = _result(top, bits)
    defect(r)
    assert _create(lib, r, _dataset(), _ends((0, 0, 0, 0, 1)), 1, 0) == (code, f"{FN}: {text}")


def _assert_slab_refusals(create, fn):
    """create(block, ends, world, rank) -> (code, message) refuses every defect of the ends table, with fn's name."""
    two = _ends((10, 20, 0, 5, 1), (30, 40, 0, 5, 1))
    assert create(_dataset(5), two, 2, 2) == (INVALID, f"{fn}: bad world or rank (0 <= rank < world <= 63)")
    assert create(_dataset(5), two, 0, 0)[1].endswith("bad world or rank (0 <= rank < world <= 63)")
    rc, msg = create(_dataset(4), two, 2, 0)
    assert rc == INVALID and msg == f"{fn}: ends_all[0] describes 5 keys, the local dataset holds 4"
    swapped = _ends((30, 40, 0, 5, 1), (10, 20, 0, 5, 1))
    rc, msg = create(_dataset(5), swapped, 2, 0)
    assert rc == INVALID and msg == f"{fn}: the slabs are out of order (rank 1's first key is below the last key of rank 0)"
    # rmi_evaluate's / rmi_train's checks of the concatenated keys, with their messages: no keys, then an unsorted slab
    assert create(_dataset(0), _ends((0, 0, 0, 0, 1), (0, 0, 0, 0, 1)), 2, 1) == \
        (PANIC, "start index was 0 but end index was 0")
    assert create(_dataset(5, sorted_=0), two, 2, 0) == (PANIC, "keys are not sorted in ascending order")


def test_refuses_bad_slabs_before_any_device_work(lib):
    r = _result(LINEAR)
    _assert_slab_refusals(lambda block, ends, world, rank: _create(lib, r, block, ends, world, rank), FN)


def test_build_refuses_bad_slabs_before_any_device_work(lib):
    _assert_slab_refusals(lambda block, ends, world, rank: _create_build(lib, block, ends, world, rank),
                          "rmi_shard_build_create")


def test_a_well_formed_result_reaches_the_dataset_checks(lib):
    rc, msg = _create(lib, _result(LINEAR), _dataset(), _ends((0, 0, 0, 0, 1)), 1, 0)
    assert rc != 0 and msg and not any(t in msg for t in SHARED_TEXTS), msg
