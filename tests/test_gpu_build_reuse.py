"""A host thread's builds share one device scratch buffer and one pinned upload slot (api.cu: BuildContext,
BuildScratch), grown to the largest build the thread has run.  Whatever ran before, a build computes what it computes
in a fresh process, bit for bit, and results of earlier builds keep their values: scratch reuse never aliases a live
result.  The sequences grow and shrink the scratch (n, N, leaf type, key type), include uint32 keys, duplicate keys,
top tables and sliced leaf launches (N >= LEAF_SLICES * 64 leaf groups of 128), and mix rmi_train, rmi_train_with_top,
rmi_train_stats_batch and rmi_evaluate on one thread and on two threads of one device at once."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from tests import datasets

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_keys(name):
    return {"u64": lambda: datasets.uniform_u64(400_000, seed=3),
            "u64_other": lambda: datasets.uniform_u64(300_000, seed=9),
            "u64_big": lambda: datasets.uniform_u64(1_500_000, seed=4),
            "u32": lambda: datasets.uniform_u32(300_000, seed=5),
            "dups": lambda: datasets.with_duplicates(datasets.uniform_u64(400_000, seed=6), 0.05),
            "small": lambda: datasets.uniform_u64(20_000, seed=7)}[name]()


# (operation, dataset, model spec or (top, [leaves]), branching factor); "evaluate" evaluates the result of
# "linear,linear" trained on `u64` with that branching factor over the named dataset
GROW_SHRINK = [
    ("train", "u64", "linear,linear", 4096),
    ("train", "u64", "linear,cubic", 100_000),         # grows; sliced leaf launch
    ("train", "u32", "radix,linear", 512),             # shrinks; uint32 keys
    ("train", "dups", "linear,linear", 65_536),        # grows; duplicate keys; sliced
    ("train", "u64_big", "linear,linear", 1 << 18),    # grows again
    ("train", "small", "cubic,linear", 256),           # shrinks
    ("train", "u64", "histogram,linear", 2048),        # top tables carved from the scratch too
    ("train", "u64_big", "linear,linear", 1 << 19),    # grows again
    ("train", "u32", "linear,linear", 40_960),         # exactly the smallest sliced launch
    ("train", "u32", "linear,linear", 40_832),         # one leaf group short of it
]
MIXED = [
    ("train", "u64", "linear,linear", 70_000),
    ("train_top", "u64", "linear,linear", 70_000),
    ("batch", "dups", ("linear", ["linear", "cubic", "linear_spline"]), 50_000),
    ("evaluate", "u64_other", "linear,linear", 70_000),
    ("train", "u64_big", "robust_linear,linear", 1 << 18),
    ("batch", "u32", ("cubic", ["linear", "loglinear"]), 1000),
]


def top_params(N):
    # a monotone linear top over [0, 2^63): x * N / 2^63
    return [0.0, float(N) / float(1 << 63)]


def snapshot(r):
    """every value of a result, copied out of the library's buffers"""
    out = {"scalars": np.array([r.model_avg_error, r.model_avg_l2_error, r.model_avg_log2_error, r.model_max_log2_error],
                               dtype=np.float64).view(np.uint64),
           "ints": np.array([r.model_max_error, r.model_max_error_idx, r.could_not_replace, r.l0_bradix_high],
                            dtype=np.uint64),
           "l0_fparams": np.array(r.l0_fparams, dtype=np.float64).view(np.uint64),
           "l0_iparams": np.array(r.l0_iparams, dtype=np.uint64)}
    for name in ("l1_params", "last_layer_max_l1s", "l1_counts", "l0_table32", "l0_radix_index", "l0_pivots"):
        a = getattr(r, name)
        if a is not None:
            out[name] = np.array(a, copy=True)
    return out


def run_op(rmi, op, data):
    """the results of one operation, as a list (a batch returns one per leaf model)"""
    kind, name, spec, N = op
    ds = data(name)
    if kind == "train":
        return [rmi.train(ds, spec, N)]
    if kind == "train_top":
        return [rmi.train(ds, spec, N, l0_params=top_params(N))]
    if kind == "batch":
        return rmi.train_stats_batch(ds, spec[0], spec[1], N)
    if kind == "evaluate":
        return [rmi.evaluate(rmi.train(data("u64"), spec, N), ds)]
    raise ValueError(kind)


def assert_same(a, b, what):
    assert sorted(a) == sorted(b), what
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, (what, k)
        assert a[k].tobytes() == b[k].tobytes(), (what, k)


def fresh_main(seq_name, index, out_path):
    """subprocess entry: one operation as the first work of a new process"""
    import rmi_b200
    rmi_b200.load_library()
    op = globals()[seq_name][index]
    cache = {}

    def data(name):
        if name not in cache:
            cache[name] = rmi_b200.RMITrainingData(make_keys(name))
        return cache[name]

    res = run_op(rmi_b200, op, data)
    np.savez(out_path, **{f"{i}/{k}": v for i, r in enumerate(res) for k, v in snapshot(r).items()})


def fresh(seq_name, index, tmp_path):
    out = str(tmp_path / f"{seq_name}_{index}.npz")
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_build_reuse as m; "
            f"m.fresh_main({seq_name!r}, {index}, {out!r})")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)
    z = np.load(out)
    res = {}
    for key in z.files:
        i, k = key.split("/", 1)
        res.setdefault(int(i), {})[k] = z[key]
    return [res[i] for i in sorted(res)]


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def data(rmi):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = rmi.RMITrainingData(make_keys(name))
        return cache[name]
    yield get
    for d in cache.values():
        d.close()


@pytest.fixture(scope="module")
def fresh_results(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("fresh")
    return {s: [fresh(s, i, tmp) for i in range(len(globals()[s]))] for s in ("GROW_SHRINK", "MIXED")}


def test_grow_shrink_matches_fresh_process(rmi, data, fresh_results):
    live, copies = [], []
    for _ in range(2):   # the second round starts from the largest buffer
        for i, op in enumerate(GROW_SHRINK):
            res = run_op(rmi, op, data)
            snaps = [snapshot(r) for r in res]
            for s, f in zip(snaps, fresh_results["GROW_SHRINK"][i]):
                assert_same(s, f, op)
            live += res
            copies += snaps
    # every result is still what it was when it was returned
    for r, s in zip(live, copies):
        assert_same(snapshot(r), s, "live result changed by a later build")


def test_mixed_entry_points_match_fresh_process(rmi, data, fresh_results):
    order = list(range(len(MIXED))) + list(reversed(range(len(MIXED)))) + [0, 4, 1, 5, 2, 3]
    live = []
    for i in order:
        res = run_op(rmi, MIXED[i], data)
        got = [snapshot(r) for r in res]
        assert len(got) == len(fresh_results["MIXED"][i])
        for s, f in zip(got, fresh_results["MIXED"][i]):
            assert_same(s, f, MIXED[i])
        live.append((i, res))
    for i, res in live:
        for r, f in zip(res, fresh_results["MIXED"][i]):
            assert_same(snapshot(r), f, ("live result changed by a later build", MIXED[i]))


def test_two_threads_on_one_device(rmi, data, fresh_results):
    ops = [("MIXED", i) for i in range(len(MIXED))] + [("GROW_SHRINK", i) for i in (1, 2, 4, 5, 8, 9)]
    for s, i in ops:   # datasets created up front, shared read-only by both threads
        data(globals()[s][i][1])
    data("u64")
    errors = []

    def worker(shift):
        try:
            seq = ops[shift:] + ops[:shift]
            for _ in range(2):
                for s, i in seq:
                    for r, f in zip(run_op(rmi, globals()[s][i], data), fresh_results[s][i]):
                        assert_same(snapshot(r), f, (s, globals()[s][i]))
        except BaseException as e:   # reported by the main thread
            errors.append(e)
        finally:
            rmi.load_library().rmi_thread_release()

    threads = [threading.Thread(target=worker, args=(k * 5,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
