"""The C ABI's consumers of a trained RMI (rmi_evaluate, rmi_index_create, rmi_index_create_bounded and
rmi_shard_index_create) run one check of the result they are given: each malformed result is refused by all four with
the same code and message, before any of them reads its dataset.  No device is needed: the dataset handle is a
zero-filled host block, which a check that read it by mistake would take for an empty dataset."""
import ctypes as C

import pytest

INVALID, UNSUPPORTED = 2, 4
N = 4                                              # leaves
LINEAR, RADIX, RADIX_TABLE, BRADIX, HISTOGRAM = 0, 7, 8, 9, 10
LEAF_TABLES = ("the result holds no leaf tables (RMI_FLAG_STATS_ONLY, or a rank other than 0 of an "
               "RMI_FLAG_SHARD_ROOT_ONLY build)")
RADIX_LEAF = "radix tables are only offered as the top model in this build"
CONSUMERS = ("rmi_evaluate", "rmi_index_create", "rmi_index_create_bounded", "rmi_shard_index_create")


@pytest.fixture(scope="module")
def lib():
    import rmi_b200
    return rmi_b200.load_library()


def _result(top=LINEAR, table_bits=0):
    """A well-formed linear-leaf result over N leaves; a radix-table top gets its table, a histogram top its pivots."""
    from rmi_b200.api import _Result
    r = _Result()
    r.num_rmi_rows = r.num_data_rows = 1000
    r.branching_factor = N
    r.l0_model_id, r.l0_table_bits = top, table_bits
    r.l1_model_id, r.l1_params_per_model = LINEAR, 2
    r.l1_params = (C.c_double * (2 * N))()
    r.l1_errors = (C.c_uint64 * N)()
    if top == RADIX_TABLE:
        r.l0_table32_len = 1 << table_bits
        r.l0_table32 = (C.c_uint32 * r.l0_table32_len)()
    if top == HISTOGRAM:
        r.l0_array2_len = 3
        r.l0_array2 = (C.c_uint64 * 3)(0, 10, 20)
    return r


def _set(**fields):
    def f(r):
        for k, v in fields.items():
            setattr(r, k, v)
    return f


def _histogram_radix_index_missing(r):
    r.l0_array1_len = 5


# (id, top, table bits, defect, code, message after "<fn>: ", a defect only for the consumers that serve error bounds)
DEFECTS = [
    ("no_leaf_params", LINEAR, 0, _set(l1_params=None), INVALID, LEAF_TABLES, False),
    ("no_leaf_errors", LINEAR, 0, _set(l1_errors=None), INVALID, LEAF_TABLES, True),
    ("unknown_top", LINEAR, 0, _set(l0_model_id=11), INVALID, "unknown model id (top 11, leaf 0)", False),
    ("unknown_leaf", LINEAR, 0, _set(l1_model_id=42), INVALID, "unknown model id (top 0, leaf 42)", False),
    ("root_only_leaf_radix", LINEAR, 0, _set(l1_model_id=RADIX), INVALID, "unknown model id (top 0, leaf 7)", False),
    ("root_only_leaf_bradix", LINEAR, 0, _set(l1_model_id=BRADIX), INVALID, "unknown model id (top 0, leaf 9)", False),
    ("root_only_leaf_histogram", LINEAR, 0, _set(l1_model_id=HISTOGRAM), INVALID, "unknown model id (top 0, leaf 10)",
     False),
    ("radix_table_width_12", RADIX_TABLE, 12, lambda r: None, INVALID, "unknown model id (top 8, leaf 0)", False),
    ("radix_table_leaf", LINEAR, 0, _set(l1_model_id=RADIX_TABLE), UNSUPPORTED, RADIX_LEAF, False),
    ("leaf_params_per_model", LINEAR, 0, _set(l1_params_per_model=3), INVALID, "wrong number of leaf parameters", False),
    ("radix_table_missing", RADIX_TABLE, 8, _set(l0_table32=None), INVALID, "radix table missing or of the wrong size",
     False),
    ("radix_table_short", RADIX_TABLE, 8, _set(l0_table32_len=255), INVALID, "radix table missing or of the wrong size",
     False),
    ("histogram_pivots_missing", HISTOGRAM, 0, _set(l0_array2=None), INVALID, "histogram pivots missing", False),
    ("histogram_pivots_empty", HISTOGRAM, 0, _set(l0_array2_len=0), INVALID, "histogram pivots missing", False),
    ("histogram_radix_index_missing", HISTOGRAM, 0, _histogram_radix_index_missing, INVALID,
     "histogram radix index missing", False),
]
SHARED_TEXTS = {d[5] for d in DEFECTS} | {"unknown model id"}


def _call(L, fn, r):
    """fn on r and an empty dataset: (return code, rmi_last_error())."""
    from rmi_b200 import api, sharded
    block = (C.c_uint64 * 8)()                       # a zero-filled rmi_dataset: no keys, never a device pointer
    ds = C.c_void_p(C.addressof(block))
    if fn == "rmi_evaluate":
        rc = L.rmi_evaluate(ds, C.byref(r), 0, C.byref(C.POINTER(api._Result)()))
    elif fn == "rmi_index_create":
        rc = L.rmi_index_create(C.byref(r), ds, C.byref(C.c_void_p()))
    elif fn == "rmi_index_create_bounded":
        knot = (C.c_uint64 * 2)(1, 0)                # one valid {key, offset}
        rc = L.rmi_index_create_bounded(C.byref(r), C.c_void_p(C.addressof(knot)), 1, 8, ds, C.byref(C.c_void_p()))
    else:
        ends = (sharded._Ends * 1)(sharded._Ends(0, 0, 0, 0, 1))   # one rank, no keys: the dataset as described
        rc = L.rmi_shard_index_create(C.byref(r), ds, ends, 1, 0, C.byref(C.c_void_p()))
    return rc, L.rmi_last_error().decode()


# rmi_evaluate re-derives the error bounds, so it accepts a result without them
CASES = [pytest.param(fn, *d[1:6], id=f"{d[0]}-{fn}") for d in DEFECTS for fn in CONSUMERS
         if not (d[6] and fn == "rmi_evaluate")]


@pytest.mark.parametrize("fn,top,bits,defect,code,text", CASES)
def test_every_consumer_refuses_a_malformed_result_alike(lib, fn, top, bits, defect, code, text):
    r = _result(top, bits)
    defect(r)
    assert _call(lib, fn, r) == (code, f"{fn}: {text}")


@pytest.mark.parametrize("fn", CONSUMERS)
@pytest.mark.parametrize("top,bits", [(LINEAR, 0), (RADIX_TABLE, 8), (RADIX_TABLE, 18), (HISTOGRAM, 0)],
                         ids=["linear", "radix8", "radix18", "histogram"])
def test_a_well_formed_result_reaches_the_dataset_checks(lib, fn, top, bits):
    """The results the defects above start from pass the shared check: each consumer refuses them for the empty
    dataset instead (an evaluation of no keys panics as the build does; the indexes find no keys or rows)."""
    rc, msg = _call(lib, fn, _result(top, bits))
    assert rc != 0 and msg
    assert not any(t in msg for t in SHARED_TEXTS), msg
