"""Host-side checks of the lookup: the table oracle (tests/lookup_oracle.py) reproduces the oracle's own lookup when
given the oracle's own tables, and rmi_index_create rejects bad arguments before touching a device."""
import ctypes as C

import numpy as np
import pytest

from tests import datasets, lookup_oracle


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    lookup_oracle.build(str(tmp_path_factory.mktemp("oracle_tables")))
    return lookup_oracle


def _queries(keys):
    if keys.dtype == np.float64:
        extra = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, np.finfo(np.float64).max], dtype=np.float64)
        return np.concatenate([keys, np.nextafter(keys, np.inf), np.nextafter(keys, -np.inf), extra])
    info = np.iinfo(keys.dtype)
    one = keys.dtype.type(1)
    extra = np.array([0, info.max], dtype=keys.dtype)
    return np.concatenate([keys, keys + one, keys - one, extra])   # wraps at the ends, as intended


CASES = [
    ("uniform_u64", "linear,linear", 1000),
    ("uniform_u64", "cubic,cubic", 500),
    ("lognormal_u64", "radix,linear_spline", 1024),
    ("uniform_u64", "radix18,robust_linear", 2000),
    ("uniform_u64", "bradix,loglinear", 256),
    ("lognormal_u64", "histogram,linear", 300),
    ("uniform_u32", "radix,normal", 512),
    ("uniform_f64", "linear,lognormal", 700),
    ("lognormal_f64", "normal,linear", 400),
    ("uniform_u64", "linear,linear", 1),
]


@pytest.mark.parametrize("dname,spec,bf", CASES)
def test_table_oracle_round_trip(oracle, tables, dname, spec, bf):
    keys = getattr(datasets, dname)(20_000)
    try:
        o = oracle.train(keys, spec, bf)
    except oracle.OraclePanic as e:
        pytest.skip(f"reference panics: {e}")
    q = _queries(keys)
    want_pos, want_err = o.lookup_batch(q)
    t = tables.from_result(o)
    pos, err = t.lookup_batch(q)
    assert np.array_equal(pos, want_pos)
    assert np.array_equal(err, want_err)


def test_index_create_rejects_bad_arguments_without_a_device():
    import rmi_b200
    from rmi_b200.api import _Result
    L = rmi_b200.load_library()
    out = C.c_void_p()
    assert L.rmi_index_create(None, None, C.byref(out)) == 2          # RMI_ERR_INVALID
    assert b"null" in L.rmi_last_error()
    r = _Result()
    r.num_rmi_rows = r.num_data_rows = 100
    r.branching_factor = 10
    r.l1_params_per_model = 2
    errors = (C.c_uint64 * 10)()
    r.l1_errors = errors                                               # l1_params stays NULL: a STATS_ONLY result
    fake_ds = C.c_void_p(1)                                            # never dereferenced: the result is refused first
    assert L.rmi_index_create(C.byref(r), fake_ds, C.byref(out)) == 2
    assert b"leaf tables" in L.rmi_last_error()
    assert L.rmi_index_create(C.byref(r), fake_ds, None) == 2
    assert not out.value
