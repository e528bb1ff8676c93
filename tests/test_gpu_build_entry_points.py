"""The C ABI's build entry points agree with one another: rmi_train, rmi_train_with_top, rmi_train_stats_batch and
rmi_shard_build_create refuse the same malformed input with the same error class and message, and a batched
statistics build reports the same top model, table sizes and statistics as the single build of each configuration."""
import ctypes as C

import numpy as np
import pytest

from tests import datasets, parity

pytestmark = pytest.mark.gpu

TOPS = ("linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal", "radix", "radix18",
        "bradix", "histogram")
LEAVES = ("linear", "cubic")
N = 1000

TWO_LAYERS = "only two-layer RMIs can be trained (the reference panics on other depths)"
RADIX_LEAF = "radix tables are only offered as the top model in this build"
NOT_SORTED = "keys are not sorted in ascending order"
BAD_BF = "branching factor must be at least 1"
BAD_TOP_PARAMS = "rmi_train_with_top: top model has no float parameters or wrong count"


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def keys():
    return datasets.uniform_u64(100_000, seed=17)


@pytest.fixture(scope="module")
def ds(rmi, keys):
    d = rmi.RMITrainingData(keys)
    yield d
    d.close()


@pytest.fixture(scope="module")
def unsorted_ds(rmi, keys):
    k = keys.copy()
    k[[10, 20]] = k[[20, 10]]
    d = rmi.RMITrainingData(k)
    yield d
    d.close()


def expect(rmi, exc, msg, fn, *args, **kw):
    """fn(*args) raises exactly `exc` (RMIPanic, or an RMIError that is not a panic) with the library's message."""
    with pytest.raises(rmi.RMIError) as info:
        fn(*args, **kw)
    assert type(info.value) is exc, (type(info.value), str(info.value))
    text = str(info.value)
    if exc is not rmi.RMIPanic:
        text = text.split(": ", 1)[1]   # "rmi_b200 error <code>: <message>"
    assert text == msg


def shard_create(rmi, data, spec, bf):
    """rmi_shard_build_create through ctypes: one rank holding the whole data set."""
    from rmi_b200 import sharded
    lib = rmi.load_library()
    lib.rmi_shard_build_create.argtypes = [C.c_void_p, C.POINTER(sharded._Ends), C.c_int, C.c_int, C.c_char_p,
                                           C.c_uint64, C.c_uint64, C.POINTER(sharded._Buffers), C.c_void_p,
                                           C.POINTER(C.c_void_p)]
    lib.rmi_shard_build_destroy.argtypes = [C.c_void_p]
    lib.rmi_shard_ends_get.argtypes = [C.c_void_p, C.POINTER(sharded._Ends)]
    ends = sharded._Ends()
    rmi.api._check(lib.rmi_shard_ends_get(data._h, C.byref(ends)))
    h = C.c_void_p()
    rc = lib.rmi_shard_build_create(data._h, C.byref(ends), 1, 0, spec.encode(), bf, 0, C.byref(sharded._Buffers()),
                                    None, C.byref(h))
    if rc == 0:
        lib.rmi_shard_build_destroy(h)
    rmi.api._check(rc)


# (spec, branching factor, unsorted data?, exception name, message)
SPEC_CASES = [
    ("bogus,linear", N, False, "RMIPanic", "Unknown model type: bogus"),
    ("linear,bogus", N, False, "RMIPanic", "Unknown model type: bogus"),
    ("linear", N, False, "RMIPanic", TWO_LAYERS),
    ("linear,linear,linear", N, False, "RMIPanic", TWO_LAYERS),
    ("linear,radix", N, False, "RMIPanic", "if used, model type radix must be the root model"),
    ("linear,bradix", N, False, "RMIPanic", "if used, model type bradix must be the root model"),
    ("linear,histogram", N, False, "RMIPanic", "if used, model type histogram must be the root model"),
    ("linear,radix18", N, False, "RMIError", RADIX_LEAF),
    ("linear,linear", 0, False, "RMIPanic", BAD_BF),
    ("linear,linear", N, True, "RMIPanic", NOT_SORTED),
]


@pytest.mark.parametrize("spec,bf,unsorted,exc,msg", SPEC_CASES)
def test_train_refuses(rmi, ds, unsorted_ds, spec, bf, unsorted, exc, msg):
    expect(rmi, getattr(rmi, exc), msg, rmi.train, unsorted_ds if unsorted else ds, spec, bf)


@pytest.mark.parametrize("spec,bf,unsorted,exc,msg", SPEC_CASES)
def test_train_with_top_refuses(rmi, ds, unsorted_ds, spec, bf, unsorted, exc, msg):
    expect(rmi, getattr(rmi, exc), msg, rmi.train, unsorted_ds if unsorted else ds, spec, bf, l0_params=[0.0, 1.0])


@pytest.mark.parametrize("spec,bf,unsorted,exc,msg", SPEC_CASES)
def test_shard_build_create_refuses(rmi, ds, unsorted_ds, spec, bf, unsorted, exc, msg):
    expect(rmi, getattr(rmi, exc), msg, shard_create, rmi, unsorted_ds if unsorted else ds, spec, bf)


@pytest.mark.parametrize("spec,bf,unsorted,exc,msg", [c for c in SPEC_CASES if c[0].count(",") == 1])
def test_stats_batch_refuses(rmi, ds, unsorted_ds, spec, bf, unsorted, exc, msg):
    top, leaf = spec.split(",")
    expect(rmi, getattr(rmi, exc), msg, rmi.train_stats_batch, unsorted_ds if unsorted else ds, top, ["linear", leaf],
           bf)


def test_train_with_top_refuses_wrong_parameters(rmi, ds):
    expect(rmi, rmi.RMIError, BAD_TOP_PARAMS, rmi.train, ds, "linear,linear", N, l0_params=[0.0, 1.0, 2.0])
    expect(rmi, rmi.RMIError, BAD_TOP_PARAMS, rmi.train, ds, "cubic,linear", N, l0_params=[0.0, 1.0])
    expect(rmi, rmi.RMIError, BAD_TOP_PARAMS, rmi.train, ds, "radix,linear", N, l0_params=[0.0, 1.0])
    expect(rmi, rmi.RMIError, BAD_TOP_PARAMS, rmi.train, ds, "radix,linear", N, l0_params=[])


STATS = ("model_max_error", "model_max_error_idx", "model_avg_error", "model_avg_l2_error", "model_avg_log2_error",
         "model_max_log2_error", "could_not_replace")


@pytest.mark.parametrize("top", TOPS)
def test_stats_batch_matches_single_builds(rmi, ds, top):
    singles = []
    for leaf in LEAVES:
        try:
            singles.append(rmi.train(ds, f"{top},{leaf}", N, counts=False))
        except rmi.RMIPanic:
            pytest.skip(f"{top},{leaf} panics on this data set")
    batch = rmi.train_stats_batch(ds, top, list(LEAVES), N)
    for leaf, g, b in zip(LEAVES, singles, batch):
        where = f"{top},{leaf}"
        assert b.l0_fparams.size == g.l0_fparams.size and b.l0_iparams.size == g.l0_iparams.size, where
        assert np.array_equal(parity.bits(b.l0_fparams), parity.bits(g.l0_fparams)), where
        assert np.array_equal(b.l0_iparams, g.l0_iparams), where
        assert b.l0_bradix_high == g.l0_bradix_high and b.l0_table_bits == g.l0_table_bits, where
        assert rmi.rmi_size(b) == rmi.rmi_size(g), where
        assert rmi.rmi_size(b, include_errors=False) == rmi.rmi_size(g, include_errors=False), where
        for f in STATS:
            assert getattr(b, f) == getattr(g, f), (where, f)
