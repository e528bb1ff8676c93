"""Range-partitioned (multi-GPU) two-layer RMI build: one process per GPU, torch.distributed
for the three small collectives, the C ABI's rmi_shard_* phases for all arithmetic.

The result is the same TrainedRMI on every rank and equals a single-GPU build of the
concatenated key array (reference semantics: rmi_lib::train on the whole data set).

    data = ShardedTrainingData(local_sorted_keys_tensor, n_local)     # rank r holds the r-th slab
    rmi  = train_sharded(data, "linear,linear", 1 << 20)

Data path per build (SURVEY.md section 8(e)):
    top model        0, 1 or 2 tiny all-reduces (TOP_ROUNDS): SUM of 8 doubles (linear /
                     robust_linear / loglinear sums; normal / lognormal mean, then variance; cubic L1
                     comparison), MIN of 4 x i64 (cubic: the two interior points of the spline);
                     or one all-reduce of the top model's table (NATIVE_ONLY_TOPS): MAX of a radix table's
                     hints or a histogram's pivots, SUM of bradix's 4 x N per-bin key counts
    all-reduce MIN   (N+1) x u64        leaf boundaries S
    (halo keys — the tail of a rank's last leaf that lives on the next rank(s) — are fetched once
     per data set, not per build: the keys are immutable)
    all-reduce SUM   N x (ppm+2) x 8 B  leaf parameters, error bounds, key counts (zero where not owned)
The orchestration below is engine-agnostic: `CudaShardEngine` drives librmi_b200.so; the
CPU tests (gloo, world_size 2) plug in a numpy engine to exercise exactly this host logic.

ShardedRMIIndex serves lookups over the same slabs (DESIGN.md section 14): a query goes to the rank whose slab holds
its lower bound, is searched there, and its global answer comes back.  ShardedBoundedRMIIndex serves a `--bounded` RMI
the same way (DESIGN.md section 17), with every rank holding only its slab of the spline's knots and a small halo.

evaluate_sharded measures a given RMI's error bounds over the same slabs (DESIGN.md section 15): every rank streams
only its own keys, and one all-reduce MAX of per-leaf maxima combines them.

cache_fix_sharded fits the `--bounded` cache-fix spline over the same slabs (DESIGN.md section 16), knot for knot the
single-GPU scan's, and train_bounded_sharded builds the bounded RMI over the knots without gathering them on one GPU.

find_pareto_efficient_configs_sharded runs the configuration search over the same slabs (DESIGN.md section 9.1): the
library's search loop, every (top, branching factor) group measured by train_stats_batch_sharded; train_for_size_sharded
is built on it.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import api

PHASE_TOP_LOCAL, PHASE_TOP_FINISH, PHASE_BOUNDS, PHASE_SPLIT, PHASE_LEAF, PHASE_STATS, PHASE_TOP_MID = range(7)
# Collectives of the top-model fit (include/rmi_b200.h rmi_shard_top_rounds): the first one follows
# TOP_LOCAL, the second one (two-round tops) follows TOP_MID.  "sum": all-reduce SUM of sums[0:8]
# as f64; "min": all-reduce MIN of sums[8:12] as signed 64-bit integers.
TOP_ROUNDS = {"linear_spline": (), "radix": (), "linear": ("sum",), "robust_linear": ("sum",), "loglinear": ("sum",),
              "normal": ("sum", "sum"), "lognormal": ("sum", "sum"), "cubic": ("min", "sum")}
# Table tops (rmi_shard_top_rounds == 4): one all-reduce of the library-owned table that rmi_shard_top_table describes
# (MAX of the hint table / the pivots, SUM of bradix's counts), between TOP_LOCAL and TOP_FINISH.  The name is older
# than the host-driven path's handle on that table; it stays bound to the code-4 tops.
NATIVE_ONLY_TOPS = ("radix8", "radix18", "radix22", "radix26", "radix28", "histogram", "bradix")
SHARDED_TOPS = tuple(TOP_ROUNDS) + NATIVE_ONLY_TOPS
TABLE_REDUCE_MAX, TABLE_REDUCE_SUM = 0, 1      # rmi_shard_top_table_info.op
_PPM = {"linear": 2, "robust_linear": 2, "linear_spline": 2, "loglinear": 2, "cubic": 4, "normal": 3, "lognormal": 3}
_TORCH_OF_KEY = {api.KEY_U64: torch.int64, api.KEY_U32: torch.int32, api.KEY_F64: torch.float64}


class _Ends(C.Structure):
    _fields_ = [("first_key_bits", C.c_uint64), ("last_key_bits", C.c_uint64), ("last_run_start", C.c_uint64),
                ("n_local", C.c_uint64), ("no_dups", C.c_uint64)]


class _TopTable(C.Structure):
    _fields_ = [("table", C.c_void_p), ("entries", C.c_uint64), ("entry_bytes", C.c_uint32), ("op", C.c_uint32)]


class _DeviceArray:
    """A 1-D view of library-owned device memory that torch.as_tensor takes without a copy."""

    def __init__(self, ptr: int, n: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


class _Buffers(C.Structure):
    _fields_ = [("sums", C.c_void_p), ("S", C.c_void_p), ("params", C.c_void_p), ("errors", C.c_void_p),
                ("counts", C.c_void_p), ("status", C.c_void_p)]


def _ends_array(ends_all: np.ndarray):
    """gather_ends' table as the C array of rmi_shard_ends that the rmi_shard_*_create calls take."""
    return (_Ends * len(ends_all))(*[_Ends(*(int(v) for v in row[:5])) for row in ends_all])


def plan_halo(bases: list[int], v: list[int], n_global: int) -> list[tuple[int, int, int, int]]:
    """v[g] = first leaf boundary S[j] >= bases[g+1] (the end of rank g's last owned leaf).
    Rank g needs global keys [bases[g+1], min(v[g] + 1, n_global)); returns the transfers
    (dst_rank, src_rank, src_local_offset, count) that deliver them."""
    world = len(bases) - 1
    moves = []
    for g in range(world - 1):
        lo, hi = bases[g + 1], min(v[g] + 1, n_global)
        for r in range(g + 1, world):
            a, b = max(lo, bases[r]), min(hi, bases[r + 1])
            if b > a:
                moves.append((g, r, a - bases[r], b - a))
    return moves


_NP_OF_KEY = {api.KEY_U64: np.uint64, api.KEY_U32: np.uint32, api.KEY_F64: np.float64}


def key_type_of_path(path: str) -> int:
    """src/main.rs:122-132: the key type is taken from the file NAME."""
    import os
    name = os.path.basename(path)
    if "uint64" in name:
        return api.KEY_U64
    if "uint32" in name:
        return api.KEY_U32
    if "f64" in name:
        return api.KEY_F64
    raise api.RMIPanic("Data file must contain uint64, uint32, or f64.")


def slab_bounds(n: int, rank: int, world: int) -> tuple[int, int]:
    """Rank r's slab of an n-key array: [n*r/world, n*(r+1)/world) — contiguous, disjoint, covering."""
    return n * rank // world, n * (rank + 1) // world


def read_slab(path: str, rank: int, world: int, key_type: int | None = None) -> tuple[np.ndarray, int]:
    """Reads ONLY this rank's slab of a reference-format key file (u64 LE count + packed keys,
    README.md:26-31 / src/load.rs:132-157) into host memory; returns (keys, total key count).
    Every rank reads 1/world of the file, so a node's ranks load the data set in parallel."""
    kt = key_type_of_path(path) if key_type is None else key_type
    dt = np.dtype(_NP_OF_KEY[kt]).newbyteorder("<")
    with open(path, "rb") as f:
        head = f.read(8)
        if len(head) != 8:
            raise api.RMIPanic(f"Unable to read the key count of {path}")
        n = int(np.frombuffer(head, dtype="<u8")[0])
        lo, hi = slab_bounds(n, rank, world)
        f.seek(8 + lo * dt.itemsize)
        keys = np.fromfile(f, dtype=dt, count=hi - lo)
    if keys.size != hi - lo:
        raise api.RMIPanic(f"{path} is shorter than its header says ({n} keys)")
    return keys.astype(_NP_OF_KEY[kt], copy=False), n


class ShardedTrainingData:
    """This rank's slab of a globally sorted key array, in device memory with room behind it
    for halo keys.  `keys` must be a 1-D torch tensor on the rank's device (int64 storage for
    uint64 keys, int32 for uint32, float64)."""

    def __init__(self, keys: torch.Tensor, n_local: int | None = None, key_type: int = api.KEY_U64,
                 halo_capacity: int = 1 << 20, group=None):
        self.group = group
        self.key_type = key_type
        n_local = keys.numel() if n_local is None else n_local
        cap = n_local + halo_capacity
        if keys.numel() >= cap:
            self.buf = keys
        else:
            self.buf = torch.empty(cap, dtype=keys.dtype, device=keys.device)
            self.buf[:n_local].copy_(keys[:n_local])
        self.n_local = n_local
        self.halo_capacity = self.buf.numel() - n_local
        self.engine = CudaShardEngine(self)

    @classmethod
    def from_file(cls, path: str, device: torch.device, key_type: int | None = None, halo_capacity: int = 1 << 20,
                  group=None) -> "ShardedTrainingData":
        """The loader of a range-partitioned build: this rank's slab of the key file -> pinned host
        memory -> its GPU (src/load.rs:132-157 for one slab)."""
        rank, world = _world(group)
        kt = key_type_of_path(path) if key_type is None else key_type
        keys, _ = read_slab(path, rank, world, kt)
        host = torch.from_numpy(keys.view(np.int64) if kt == api.KEY_U64 else (keys.view(np.int32) if kt == api.KEY_U32 else keys))
        if torch.cuda.is_available():
            host = host.pin_memory()
        dev_keys = torch.empty(host.numel() + halo_capacity, dtype=host.dtype, device=device)
        dev_keys[: host.numel()].copy_(host, non_blocking=False)
        return cls(dev_keys, host.numel(), kt, halo_capacity, group)

    def grow_halo(self, capacity: int):
        """Re-home the slab in a buffer with room for `capacity` halo keys (a leaf reached further
        into the following ranks than expected — heavy skew)."""
        old = self.buf
        self.buf = torch.empty(self.n_local + capacity, dtype=old.dtype, device=old.device)
        self.buf[: self.n_local].copy_(old[: self.n_local])
        self.halo_capacity = capacity
        self.engine.end()
        self.engine = CudaShardEngine(self)
        for attr in ("_min_cap", "_halo_have"):
            if hasattr(self, attr):
                delattr(self, attr)


class CudaShardEngine:
    """Phases of a range-partitioned build on librmi_b200.so (include/rmi_b200.h rmi_shard_*)."""

    def __init__(self, data: ShardedTrainingData):
        self.data = data
        self.lib = api.load_library()
        L = self.lib
        L.rmi_shard_ends_get.argtypes = [C.c_void_p, C.POINTER(_Ends)]
        L.rmi_shard_build_create.argtypes = [C.c_void_p, C.POINTER(_Ends), C.c_int, C.c_int, C.c_char_p, C.c_uint64,
                                             C.c_uint64, C.POINTER(_Buffers), C.c_void_p, C.POINTER(C.c_void_p)]
        L.rmi_shard_phase.argtypes = [C.c_void_p, C.c_int]
        L.rmi_shard_set_halo.argtypes = [C.c_void_p, C.c_uint64]
        L.rmi_shard_top_table.argtypes = [C.c_void_p, C.POINTER(_TopTable)]
        L.rmi_shard_finish.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.POINTER(api._Result))]
        L.rmi_shard_build_destroy.argtypes = [C.c_void_p]
        L.rmi_shard_comm_unique_id.argtypes = [C.c_void_p]
        L.rmi_shard_comm_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.rmi_shard_comm_destroy.argtypes = [C.c_void_p]
        L.rmi_shard_train.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.POINTER(api._Result))]
        L.rmi_shard_stats_batch_create.argtypes = [C.c_void_p, C.POINTER(_Ends), C.c_int, C.c_int, C.c_char_p,
                                                   C.POINTER(C.c_char_p), C.c_int, C.c_uint64, C.c_uint64, C.POINTER(_Buffers),
                                                   C.c_void_p, C.POINTER(C.c_void_p)]
        L.rmi_shard_stats_leaf.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.rmi_shard_stats_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.POINTER(api._Result))]
        L.rmi_shard_train_stats_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.POINTER(api._Result))]
        self.device = data.buf.device
        self.ds = api.RMITrainingData.from_device(data.buf.data_ptr(), data.n_local, data.key_type,
                                                  self.device.index or 0, keep_alive=data.buf)
        self._build = None

    def ends(self):
        e = _Ends()
        api._check(self.lib.rmi_shard_ends_get(self.ds._h, C.byref(e)))
        return int(e.first_key_bits), int(e.last_key_bits), int(e.last_run_start), int(e.n_local), int(e.no_dups)

    def begin(self, ends_all: np.ndarray, world: int, rank: int, spec: str, num_leaves: int, bufs: dict):
        key = (spec, num_leaves, tuple(bufs[k].data_ptr() for k in sorted(bufs)))
        if self._build is not None and getattr(self, "_build_key", None) == key:
            return      # same spec / buffers: the build object (scratch, events) is reused
        self.end()
        self._build_key = key
        cb = _Buffers(*(bufs[k].data_ptr() for k in ("sums", "S", "params", "errors", "counts", "status")))
        h = C.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        api._check(self.lib.rmi_shard_build_create(self.ds._h, _ends_array(ends_all), world, rank, spec.encode(),
                                                   num_leaves, self.data.halo_capacity, C.byref(cb), C.c_void_p(stream),
                                                   C.byref(h)))
        self._build = h
        self._spec = spec

    def begin_batch(self, ends_all: np.ndarray, world: int, rank: int, top: str, leaves: list[str], num_leaves: int, bufs: dict):
        """A statistics-only batch of the leaf types `leaves` under one top model (rmi_shard_stats_batch_create)."""
        key = ("batch", top, tuple(leaves), num_leaves, tuple(bufs[k].data_ptr() for k in sorted(bufs)))
        if self._build is not None and getattr(self, "_build_key", None) == key:
            return
        self.end()
        self._build_key = key
        cb = _Buffers(*(bufs[k].data_ptr() for k in ("sums", "S", "params", "errors", "counts", "status")))
        names = (C.c_char_p * len(leaves))(*[m.encode() for m in leaves])
        h = C.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        api._check(self.lib.rmi_shard_stats_batch_create(self.ds._h, _ends_array(ends_all), world, rank, top.encode(), names,
                                                         len(leaves), num_leaves, self.data.halo_capacity, C.byref(cb),
                                                         C.c_void_p(stream), C.byref(h)))
        self._build = h
        self._batch = [f"{top},{m}" for m in leaves]

    def stats_leaf(self, k: int, record: torch.Tensor):
        """Leaf type k of the batch over the leaves this rank owns: its record (STATS_RECORD_WORDS int64) into `record`."""
        api._check(self.lib.rmi_shard_stats_leaf(self._build, int(k), C.c_void_p(record.data_ptr())))

    def stats_finish(self, records: torch.Tensor, flags: int = 0):
        """The batch's results from every rank's records (world x K records, rank by rank, on this device)."""
        out = (C.POINTER(api._Result) * len(self._batch))()
        api._check(self.lib.rmi_shard_stats_finish(self._build, C.c_void_p(records.data_ptr()), int(flags), out))
        return [api.result_from_pointer(out[k], spec) for k, spec in enumerate(self._batch)]

    def train_stats_batch(self, comm, flags: int = 0):
        """The whole batch in one library call (rmi_shard_train_stats_batch)."""
        out = (C.POINTER(api._Result) * len(self._batch))()
        api._check(self.lib.rmi_shard_train_stats_batch(self._build, comm, int(flags), out))
        return [api.result_from_pointer(out[k], spec) for k, spec in enumerate(self._batch)]

    def phase(self, k: int):
        api._check(self.lib.rmi_shard_phase(self._build, k))

    def set_halo(self, count: int):
        api._check(self.lib.rmi_shard_set_halo(self._build, count))

    def top_table(self):
        """(table, op) of a code-4 top model (rmi_shard_top_table): an int32 / int64 device view of the u32 / u64
        entries and TABLE_REDUCE_MAX / _SUM; None for the other tops."""
        t = _TopTable()
        api._check(self.lib.rmi_shard_top_table(self._build, C.byref(t)))
        if t.entries == 0:
            return None
        typestr = "<i4" if t.entry_bytes == 4 else "<i8"
        return torch.as_tensor(_DeviceArray(int(t.table), int(t.entries), typestr), device=self.device), int(t.op)

    def halo_view(self, offset: int, count: int) -> torch.Tensor:
        n = self.data.n_local
        return self.data.buf[n + offset: n + offset + count]

    def local_view(self, offset: int, count: int) -> torch.Tensor:
        return self.data.buf[offset: offset + count]

    def train(self, comm, flags: int = 0):
        """The whole build in one library call: phases and NCCL collectives on the build's stream (rmi_shard_train)."""
        res = C.POINTER(api._Result)()
        api._check(self.lib.rmi_shard_train(self._build, comm, int(flags), C.byref(res)))
        return api.result_from_pointer(res, self._spec)

    def finish(self, flags: int = 0):
        res = C.POINTER(api._Result)()
        api._check(self.lib.rmi_shard_finish(self._build, int(flags), C.byref(res)))
        return api.result_from_pointer(res, self._spec)

    def lookup_index(self, trained, ends_all: np.ndarray, world: int, rank: int) -> "CudaShardIndex":
        return CudaShardIndex(self, trained, ends_all, world, rank)

    def bounded_lookup_index(self, trained, knots: np.ndarray, halo_before: int, knot_counts: list[int], line_size: int,
                             ends_all: np.ndarray, world: int, rank: int) -> "CudaShardBoundedIndex":
        return CudaShardBoundedIndex(self, trained, knots, halo_before, knot_counts, line_size, ends_all, world, rank)

    def evaluator(self, trained, ends_all: np.ndarray, world: int, rank: int) -> "CudaShardEval":
        return CudaShardEval(self, trained, ends_all, world, rank)

    def cache_fixer(self, ends_all: np.ndarray, world: int, rank: int, line_size: int, halo_keys: int) -> "CudaShardCacheFix":
        return CudaShardCacheFix(self, ends_all, world, rank, line_size, halo_keys)

    def end(self):
        if self._build is not None:
            self.lib.rmi_shard_build_destroy(self._build)
            self._build = None

    def __del__(self):
        try:
            self.end()
        except Exception:
            pass


def _world(group):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


_native_comms = {}


def native_comm(group, device: torch.device, single_rank_ok: bool = False):
    """The library's own NCCL communicator for `group` (rmi_shard_comm_*): rank 0 draws the unique id, the
    128 bytes travel through torch.distributed, every rank joins.  Cached per (group, device).  Returns None
    when the group does not run over NCCL (gloo tests; a single rank unless single_rank_ok — a one-rank
    communicator is how the one-call path is exercised on a one-GPU box) or NCCL cannot be loaded."""
    rank, world = _world(group)
    if device.type != "cuda" or (world > 1 and dist.get_backend(group) != "nccl") or (world <= 1 and not single_rank_ok):
        return None
    key = (id(group) if group is not None else 0, device.index or 0, world)
    if key in _native_comms:
        return _native_comms[key]
    lib = api.load_library()
    lib.rmi_shard_comm_unique_id.argtypes = [C.c_void_p]
    lib.rmi_shard_comm_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    buf = (C.c_uint8 * 128)()
    ok = 1
    if rank == 0:
        ok = 1 if lib.rmi_shard_comm_unique_id(buf) == 0 else 0
    if world > 1:
        t = torch.tensor(list(buf) + [ok], dtype=torch.uint8, device=device)
        dist.broadcast(t, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        vals = t.cpu().tolist()
    else:
        vals = list(buf) + [ok]
    comm = None
    if vals[128] == 1:
        ident = (C.c_uint8 * 128)(*vals[:128])
        h = C.c_void_p()
        api._check(lib.rmi_shard_comm_create(ident, world, rank, device.index or 0, C.byref(h)))
        comm = h
    _native_comms[key] = comm
    return comm


def gather_ends(data, eng, group) -> np.ndarray:
    """Every rank's rmi_shard_ends (first / last key bits, last run start, n_local, no_dups) as a (world, 5) uint64
    array, identical on every rank.  Collective on the first call; cached on `data` (the keys are immutable)."""
    ends_all = getattr(data, "_ends_all", None)
    if ends_all is None:
        rank, world = _world(group)
        e = torch.tensor(np.array(eng.ends(), dtype=np.uint64).view(np.int64), dtype=torch.int64, device=eng.device)
        gathered = [torch.empty_like(e) for _ in range(world)]
        if world > 1:
            dist.all_gather(gathered, e, group=group)
        else:
            gathered = [e]
        ends_all = torch.stack(gathered).cpu().numpy().view(np.uint64)
        data._ends_all = ends_all
    return ends_all


def train_sharded(data, model_spec: str, num_leaves: int, flags: int = 0, group=None, engine=None, counts: bool = True,
                  native: bool | None = None):
    """rmi_lib::train on a range-partitioned key array; returns the full TrainedRMI on every rank.

    native=None (default): with the CUDA engine over an NCCL group the whole build is ONE library call
    (rmi_shard_train: kernels and collectives on one stream, leaf records exchanged as an all-gather by
    ownership range); otherwise — gloo, the numpy engine of the CPU tests, native=False — the phases are
    sequenced here and the collectives go through torch.distributed."""
    eng = engine if engine is not None else data.engine
    group = group if group is not None else getattr(data, "group", None)
    rank, world = _world(group)
    dev = eng.device
    parts = model_spec.split(",")
    if len(parts) != 2:
        raise api.RMIPanic("only two-layer RMIs can be trained (the reference panics on other depths)")
    if parts[0] not in SHARDED_TOPS:
        raise api.RMIError(f"range-partitioned builds offer the top models {SHARDED_TOPS}")
    ppm = _PPM.get(parts[1])
    if ppm is None:
        raise api.RMIPanic(f"unsupported or unknown leaf model {parts[1]}")
    N = int(num_leaves)

    # 1. what every rank's slab looks like at its ends (cached on the data object: the data is immutable)
    ends_all = gather_ends(data, eng, group)
    bases = [0]
    for n_local in ends_all[:, 3]:
        bases.append(bases[-1] + int(n_local))
    n_global = bases[-1]

    bufs = _buffers(data, N, ppm, dev)
    eng.begin(ends_all, world, rank, model_spec, N, bufs)

    comm = None
    if native is not False and isinstance(eng, CudaShardEngine):
        comm = native_comm(group, dev, single_rank_ok=native is True)
        if native is True and comm is None:
            raise api.RMIError("native=True needs an NCCL process group (or a single rank) and a loadable libnccl.so.2")
    if comm is not None:
        # halo keys are fetched once per data set (see step 4 below), then the whole build is one call
        _fetch_halo_once(data, eng, bases, n_global, group, world, rank, dev)
        try:
            return eng.train(comm, int(flags) | (api.FLAG_LEAF_COUNTS if counts else 0))
        except api.RMIPanic as e:
            if "halo" not in str(e):
                raise
        return _retry_with_larger_halo(data, bufs, bases, n_global, N, model_spec, num_leaves, flags, group, world, dev, counts, native)

    _host_top_and_bounds(data, eng, bufs, parts[0], bases, n_global, group, world, rank, dev)
    # 5. leaves owned by this rank, then everyone gets everything
    eng.phase(PHASE_LEAF)
    if world > 1:
        rec = bufs["records"]
        dist.all_reduce(rec if counts else rec[: N * (ppm + 1)], op=dist.ReduceOp.SUM, group=group)
        # the status word is a BIT MASK (kernels.h StatusBit): combine by OR, not MAX, so that every rank sees every
        # rank's bits and all of them take the same decision below (retry with a larger halo / raise)
        st_all = [torch.empty_like(bufs["status"]) for _ in range(world)]
        dist.all_gather(st_all, bufs["status"], group=group)
        acc = st_all[0].clone()
        for t in st_all[1:]:
            acc |= t
        bufs["status"].copy_(acc)
    eng.phase(PHASE_STATS)
    try:
        return eng.finish(int(flags) | (api.FLAG_LEAF_COUNTS if counts else 0))
    except api.RMIPanic as e:
        if world <= 1 or "halo" not in str(e):
            raise
    return _retry_with_larger_halo(data, bufs, bases, n_global, N, model_spec, num_leaves, flags, group, world, dev, counts, native)


def _buffers(data, N: int, ppm: int, dev) -> dict:
    """The device buffers of a build of N leaves with ppm parameters per leaf (cached on `data`)."""
    bufs = getattr(data, "_bufs", None)
    if bufs is None or bufs["S"].numel() != N + 1 or bufs["params"].numel() != N * ppm:
        # params | errors | counts live in ONE allocation so that a single all-reduce combines them
        rec = torch.empty(N * (ppm + 2), dtype=torch.int64, device=dev)
        bufs = dict(sums=torch.zeros(16, dtype=torch.float64, device=dev),   # [0:8] f64 sums, [8:16] i64 slots
                    S=torch.empty(N + 1, dtype=torch.int64, device=dev),
                    params=rec[: N * ppm].view(torch.float64),
                    errors=rec[N * ppm: N * (ppm + 1)],
                    counts=rec[N * (ppm + 1):],
                    status=torch.zeros(1, dtype=torch.int32, device=dev), records=rec)
        data._bufs = bufs
    return bufs


def _fetch_halo_once(data, eng, bases, n_global, group, world, rank, dev):
    """The first halo_capacity keys behind every slab, fetched once per data set (the keys are immutable)."""
    if getattr(data, "_halo_have", None) is None:
        if world > 1:
            cap = _min_halo_capacity(data, group, world, dev)
            moves = plan_halo(bases, [bases[g + 1] + cap - 1 for g in range(world)], n_global)
            data._halo_have = _exchange_halo(eng, moves, rank, group, dev)
        else:
            data._halo_have = 0
    eng.set_halo(data._halo_have or 0)


def _host_top_and_bounds(data, eng, bufs, top, bases, n_global, group, world, rank, dev):
    """Host-sequenced phases of a build up to the leaves: the top model with its collectives, the leaf boundaries
    with their all-reduce MIN, the split, and the halo."""
    # 2. top model: local part -> tiny all-reduce(s) -> closed form (identical on every rank)
    def top_collective(kind):
        if world <= 1:
            return
        if kind == "sum":
            dist.all_reduce(bufs["sums"][:8], op=dist.ReduceOp.SUM, group=group)
        else:
            dist.all_reduce(bufs["sums"].view(torch.int64)[8:12], op=dist.ReduceOp.MIN, group=group)

    rounds = TOP_ROUNDS.get(top, ())
    eng.phase(PHASE_TOP_LOCAL)
    if top in NATIVE_ONLY_TOPS and world > 1:
        table = eng.top_table()
        if table is not None:
            # gloo cannot reduce device memory (one-GPU test boxes): stage through the host there
            _merge_top_table(*table, group, dev.type == "cuda" and dist.get_backend(group) == "gloo")
    if rounds:
        top_collective(rounds[0])
    if len(rounds) > 1:
        eng.phase(PHASE_TOP_MID)
        top_collective(rounds[1])
    eng.phase(PHASE_TOP_FINISH)
    # 3. leaf boundaries: local lower bounds -> all-reduce MIN
    eng.phase(PHASE_BOUNDS)
    if world > 1:
        dist.all_reduce(bufs["S"], op=dist.ReduceOp.MIN, group=group)
    eng.phase(PHASE_SPLIT)
    # 4. halo: the keys of a rank's last leaf that live on the following rank(s).  The keys are
    #    immutable, so the first `halo_capacity` keys behind every slab are fetched ONCE per data set
    #    (no planning, no host synchronisation, no transfer inside a build); a build whose last leaf
    #    reaches further reports it through the status word and takes the planned path below.
    if world > 1 and getattr(data, "_halo_have", None) is None:
        cap = _min_halo_capacity(data, group, world, dev)
        moves = plan_halo(bases, [bases[g + 1] + cap - 1 for g in range(world)], n_global)
        data._halo_have = _exchange_halo(eng, moves, rank, group, dev)
    eng.set_halo(getattr(data, "_halo_have", 0) or 0)


def _merge_top_table(table: torch.Tensor, op: int, group, stage: bool):
    """All-reduce, in place, of a code-4 top model's table: `table` is the signed torch view (int32 / int64) of its
    unsigned entries.  torch reduces signed integers, so MAX runs on the entries with their sign bit flipped (signed
    order == unsigned order), and the u32 counts of a SUM are added as int64 and wrapped back to 32 bits."""
    if op == TABLE_REDUCE_SUM:
        assert table.dtype == torch.int32
        h = table.to(torch.int64) & 0xFFFFFFFF
        h = h.cpu() if stage else h
        dist.all_reduce(h, op=dist.ReduceOp.SUM, group=group)
        h = h & 0xFFFFFFFF
        table.copy_(torch.where(h >= 1 << 31, h - (1 << 32), h).to(torch.int32))
    else:
        sign = -(1 << (8 * table.element_size() - 1))
        h = table ^ sign
        h = h.cpu() if stage else h
        dist.all_reduce(h, op=dist.ReduceOp.MAX, group=group)
        table.copy_(h ^ sign)


def evaluate_sharded(trained, data, flags: int = 0, group=None, engine=None, counts: bool = True,
                     native: bool | None = None):
    """api.evaluate of ``trained``'s tables over a range-partitioned key array (DESIGN.md section 15): the error bounds,
    key counts (counts=True) and statistics of the concatenated slabs, bit for bit, on every rank; the tables are
    returned unchanged.  Each rank reads only its own keys.  Raises RMIPanic on every rank where the top model is not
    monotone on the keys (a cut included).

    native=None (default): with the CUDA engine over an NCCL group it is ONE library call (rmi_shard_evaluate);
    otherwise (gloo, a numpy engine, native=False) the phases are driven here: bounds -> all-reduce MIN of S -> keys ->
    all-reduce MAX of the partial maxima and an all-gather of the status words -> finish."""
    eng = engine if engine is not None else data.engine
    group = group if group is not None else getattr(data, "group", None)
    rank, world = _world(group)
    dev = eng.device
    flags = int(flags) | (api.FLAG_LEAF_COUNTS if counts else 0)
    ev = eng.evaluator(trained, gather_ends(data, eng, group), world, rank)
    try:
        comm = None
        if native is not False and isinstance(ev, CudaShardEval):
            comm = native_comm(group, dev, single_rank_ok=native is True)
            if native is True and comm is None:
                raise api.RMIError("native=True needs an NCCL process group (or a single rank) and a loadable libnccl.so.2")
        if comm is not None:
            return ev.evaluate(comm, flags)
        # gloo cannot reduce device memory (one-GPU test boxes): stage through the host there
        stage = world > 1 and dev.type == "cuda" and dist.get_backend(group) == "gloo"

        def all_reduce(t, op):
            if world <= 1:
                return
            h = t.cpu() if stage else t
            dist.all_reduce(h, op=op, group=group)
            if stage:
                t.copy_(h)

        S = ev.bounds()
        all_reduce(S, dist.ReduceOp.MIN)
        part, status = ev.keys(S)
        all_reduce(part[: ev.partial_words], dist.ReduceOp.MAX)
        # the status word is a BIT MASK: every rank ORs every rank's word, so that all of them fail alike
        st = status.cpu() if stage else status
        st_all = [torch.empty_like(st) for _ in range(world)]
        if world > 1:
            dist.all_gather(st_all, st, group=group)
        else:
            st_all = [st]
        acc = 0
        for t in st_all:
            acc |= int(t[0]) & 0xFFFFFFFF
        return ev.finish(S, part, acc, flags)
    finally:
        ev.close()


def _retry_with_larger_halo(data, bufs, bases, n_global, N, model_spec, num_leaves, flags, group, world, dev, counts, native):
    # A leaf reaches past the prefetched halo (heavy skew).  The status word is the OR over ranks, so
    # every rank arrives here together: size the halo from the global boundaries S and build again.
    _grow_halo(data, bufs, bases, n_global, N, group, world, dev)
    return train_sharded(data, model_spec, num_leaves, flags, group, counts=counts, native=native)


def _grow_halo(data, bufs, bases, n_global, N, group, world, dev):
    """Re-home every slab behind a halo that holds the keys the boundaries S of the last build need (collective)."""
    S = bufs["S"]
    cuts = torch.tensor(bases[1:], dtype=torch.int64, device=dev)
    pos = torch.searchsorted(S, cuts).clamp_(max=N)
    v = S[pos].cpu().tolist()
    need = {}
    for (dst, src, off, cnt) in plan_halo(bases, v, n_global):
        need[dst] = need.get(dst, 0) + cnt
    most = max(need.values(), default=0)
    if most <= _min_halo_capacity(data, group, world, dev) or not hasattr(data, "grow_halo"):
        raise api.RMIError(f"a leaf reaches further into the next rank than the halo capacity ({most} keys needed)")
    data.grow_halo(int(most * 1.25) + 1024)


STATS_RECORD_WORDS = 6      # RMI_SHARD_STATS_RECORD_BYTES / 8: a rank's statistics partial and status words of one leaf type


def train_stats_batch_sharded(data, top_model: str, leaf_models: list[str], num_leaves: int, flags: int = 0, group=None,
                              engine=None, native: bool | None = None) -> list:
    """api.train_stats_batch over a range-partitioned key array (DESIGN.md section 9): the statistics-only results of
    "top_model,leaf" for every leaf of `leaf_models` at `num_leaves` leaves, the same list on every rank.  The top
    model and the leaf boundaries are derived once; every rank fits only the leaves it owns, for every leaf type, and
    one all-gather of K x 48 bytes per rank carries the statistics.  No result holds leaf tables.

    native=None (default): with the CUDA engine over an NCCL group the batch is ONE library call
    (rmi_shard_train_stats_batch); otherwise (gloo, the numpy engine, native=False) the phases are sequenced here.  A leaf
    that reaches past the halo grows the halo (it never shrinks) and measures the batch again."""
    eng = engine if engine is not None else data.engine
    group = group if group is not None else getattr(data, "group", None)
    rank, world = _world(group)
    dev = eng.device
    if top_model not in SHARDED_TOPS:
        raise api.RMIError(f"range-partitioned builds offer the top models {SHARDED_TOPS}")
    leaves = list(leaf_models)
    if not leaves:
        raise api.RMIError("train_stats_batch_sharded: no leaf models")
    N = int(num_leaves)
    ends_all = gather_ends(data, eng, group)
    bases = [0]
    for n_local in ends_all[:, 3]:
        bases.append(bases[-1] + int(n_local))
    n_global = bases[-1]
    # the batch reads S, the sums, the error bounds, the counts and the status word; its leaf parameters go to its own
    # scratch, so the buffers of a two-parameter leaf do for every leaf type
    bufs = _buffers(data, N, _PPM.get(leaves[0], 2), dev)
    eng.begin_batch(ends_all, world, rank, top_model, leaves, N, bufs)
    comm = None
    if native is not False and isinstance(eng, CudaShardEngine):
        comm = native_comm(group, dev, single_rank_ok=native is True)
        if native is True and comm is None:
            raise api.RMIError("native=True needs an NCCL process group (or a single rank) and a loadable libnccl.so.2")
    try:
        if comm is not None:
            _fetch_halo_once(data, eng, bases, n_global, group, world, rank, dev)
            return eng.train_stats_batch(comm, int(flags))
        _host_top_and_bounds(data, eng, bufs, top_model, bases, n_global, group, world, rank, dev)
        K = len(leaves)
        mine = torch.empty(K * STATS_RECORD_WORDS, dtype=torch.int64, device=dev)
        for k in range(K):
            eng.stats_leaf(k, mine[k * STATS_RECORD_WORDS:(k + 1) * STATS_RECORD_WORDS])
        if world > 1:
            # gloo cannot gather device memory (one-GPU test boxes): stage through the host there
            stage = dev.type == "cuda" and dist.get_backend(group) == "gloo"
            src = mine.cpu() if stage else mine
            got = [torch.empty_like(src) for _ in range(world)]
            dist.all_gather(got, src, group=group)
            records = torch.cat(got).to(dev)
        else:
            records = mine
        return eng.stats_finish(records, int(flags))
    except api.RMIPanic as e:
        if world <= 1 or "halo" not in str(e):
            raise
    _grow_halo(data, bufs, bases, n_global, N, group, world, dev)
    return train_stats_batch_sharded(data, top_model, leaves, num_leaves, flags, group, native=native)


_MEASURE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_char_p, C.c_uint64, C.POINTER(C.c_char_p), C.c_int, C.c_uint32,
                          C.POINTER(api._ConfigStats))


def find_pareto_efficient_configs_sharded(data, restrict_to: int = 10, flags: int = 0, group=None, native: bool | None = None,
                                          engine=None) -> list[dict]:
    """api.find_pareto_efficient_configs over a range-partitioned key array.  Collective: every rank calls it and every
    rank returns the same list.  The search itself is the library's (host/optimizer.hpp, rmi_find_pareto_efficient_configs_with),
    run on every rank over bit-identical merged statistics, so no rank coordinates the others; each (top model,
    branching factor) group is measured by train_stats_batch_sharded.  RMI_OPTIMIZER_PROFILE selects the grid."""
    L = api.load_library()
    L.rmi_find_pareto_efficient_configs_with.argtypes = [_MEASURE_FN, C.c_void_p, C.c_uint64, C.c_uint32,
                                                         C.POINTER(api._ConfigStats), C.c_uint64, C.POINTER(C.c_uint64)]
    failures = []

    def measure(_ctx, top, bf, leaves, k_count, fl, out):
        try:
            names = [leaves[k].decode() for k in range(k_count)]
            res = train_stats_batch_sharded(data, top.decode(), names, int(bf), int(fl), group=group, engine=engine,
                                            native=native)
            for k, r in enumerate(res):
                out[k].average_log2_error = r.model_avg_log2_error
                out[k].max_log2_error = r.model_max_log2_error
                out[k].size = api.rmi_size(r)
            return 0
        except BaseException as e:  # noqa: BLE001 - re-raised below, after the library has unwound the search
            failures.append(e)
            return 1

    cb = _MEASURE_FN(measure)
    cap = max(4096, int(restrict_to) if restrict_to < (1 << 20) else 0)
    out = (api._ConfigStats * cap)()
    cnt = C.c_uint64(0)
    rc = L.rmi_find_pareto_efficient_configs_with(cb, None, int(restrict_to), int(flags), out, cap, C.byref(cnt))
    if failures:
        raise failures[0]
    api._check(rc)
    if int(cnt.value) > cap:
        raise api.RMIError(f"Pareto front has {int(cnt.value)} entries, more than the {cap} this call can return")
    return [dict(models=out[i].models.decode(), branching_factor=int(out[i].branching_factor),
                 average_log2_error=float(out[i].average_log2_error), max_log2_error=float(out[i].max_log2_error),
                 size=int(out[i].size)) for i in range(int(cnt.value))]


def train_for_size_sharded(data, max_size: int, flags: int = 0, group=None, native: bool | None = None):
    """api.train_for_size over a range-partitioned key array (collective): the first configuration of the un-narrowed
    Pareto front smaller than max_size bytes, trained with train_sharded."""
    front = find_pareto_efficient_configs_sharded(data, 1000, flags, group=group, native=native)
    pick = next((c for c in front if c["size"] < max_size), None)
    if pick is None:
        raise api.RMIPanic(f"Could not find any configurations smaller than {max_size}")
    return train_sharded(data, pick["models"], pick["branching_factor"], flags, group, native=native)


def _exchange_halo(eng, moves, rank, group, dev) -> int:
    """Carries out plan_halo's transfers; returns how many halo keys this rank now holds."""
    # gloo cannot send/recv device memory (one-GPU test boxes): stage through the host there
    stage = dev.type == "cuda" and dist.get_backend(group) == "gloo"
    ops, recv_off, landed = [], 0, []
    for (dst, src, off, cnt) in moves:
        if dst == rank:
            view = eng.halo_view(recv_off, cnt)
            t = torch.empty(cnt, dtype=view.dtype) if stage else view
            if stage:
                landed.append((view, t))
            ops.append(dist.P2POp(dist.irecv, t, src, group=group))
            recv_off += cnt
        elif src == rank:
            view = eng.local_view(off, cnt)
            ops.append(dist.P2POp(dist.isend, view.cpu() if stage else view, dst, group=group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    for view, t in landed:
        view.copy_(t)
    return recv_off


def _min_halo_capacity(data, group, world, dev):
    cap = getattr(data, "_min_cap", None)
    if cap is None:
        t = torch.tensor([data.halo_capacity], dtype=torch.int64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
        cap = int(t.item())
        data._min_cap = cap
    return cap


# ---- lookups over the slabs (include/rmi_b200.h rmi_shard_index_*, DESIGN.md section 14) ------------------------------

class _LookupStats(C.Structure):
    _fields_ = [("phase_ms", C.c_float * 6), ("queries_routed", C.c_uint64), ("queries_searched", C.c_uint64),
                ("queries_kept", C.c_uint64)]


LOOKUP_PHASES = ("route", "count_exchange", "query_exchange", "search", "answer_exchange", "gather")


class CudaShardIndex:
    """One rank's side of the lookups over the slabs on librmi_b200.so (rmi_shard_index_*).  Every call enqueues on
    the current torch stream of the data's device and returns device tensors."""

    def __init__(self, eng: CudaShardEngine, trained, ends_all: np.ndarray, world: int, rank: int):
        L = self._bind(eng, trained, world)
        api._check(L.rmi_shard_index_create(api._result_ptr(trained), eng.ds._h, _ends_array(ends_all), world, rank,
                                            C.byref(self._h)))

    def _bind(self, eng: CudaShardEngine, trained, world: int):
        L = self.lib = api.load_library()
        L.rmi_shard_index_create.argtypes = [C.POINTER(api._Result), C.c_void_p, C.POINTER(_Ends), C.c_int, C.c_int,
                                             C.POINTER(C.c_void_p)]
        L.rmi_shard_index_destroy.argtypes = [C.c_void_p]
        L.rmi_shard_index_predict.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_shard_index_route.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
        L.rmi_shard_index_search.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_shard_index_gather.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        L.rmi_shard_index_lower_bound.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                                  C.c_void_p, C.c_void_p]
        L.rmi_shard_index_last_stats.argtypes = [C.c_void_p, C.POINTER(_LookupStats)]
        L.rmi_shard_index_route_upper.argtypes = L.rmi_shard_index_route.argtypes
        L.rmi_shard_index_search_upper.argtypes = L.rmi_shard_index_search.argtypes
        L.rmi_shard_index_upper_bound.argtypes = L.rmi_shard_index_lower_bound.argtypes
        self.device = eng.device
        self.world = world
        self._ds = eng.ds            # the slab the index searches: kept alive with it
        self._trained = trained
        self._h = C.c_void_p()
        return L

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream or None)

    def _u64(self, n: int) -> torch.Tensor:
        return torch.empty(n, dtype=torch.int64, device=self.device)

    def predict(self, q: torch.Tensor):
        pos, err = self._u64(q.numel()), self._u64(q.numel())
        api._check(self.lib.rmi_shard_index_predict(self._h, q.data_ptr(), q.numel(), pos.data_ptr(), err.data_ptr(),
                                                    self._stream()))
        return pos, err

    def route(self, q: torch.Tensor, fn=None):
        send, slot, counts = torch.empty_like(q), self._u64(q.numel()), self._u64(self.world)
        api._check((fn or self.lib.rmi_shard_index_route)(self._h, q.data_ptr(), q.numel(), send.data_ptr(),
                                                          slot.data_ptr(), counts.data_ptr(), self._stream()))
        return send, slot, counts

    def search(self, recv: torch.Tensor, fn=None):
        answers, fb = self._u64(recv.numel()), torch.zeros(1, dtype=torch.int64, device=self.device)
        api._check((fn or self.lib.rmi_shard_index_search)(self._h, recv.data_ptr(), recv.numel(), answers.data_ptr(),
                                                           fb.data_ptr(), self._stream()))
        return answers, fb

    def route_upper(self, q: torch.Tensor):
        """route by <= (the upper bound's rule)"""
        return self.route(q, self.lib.rmi_shard_index_route_upper)

    def search_upper(self, recv: torch.Tensor):
        return self.search(recv, self.lib.rmi_shard_index_search_upper)

    def gather(self, slot: torch.Tensor, returned: torch.Tensor):
        out = self._u64(slot.numel())
        api._check(self.lib.rmi_shard_index_gather(self._h, slot.data_ptr(), returned.data_ptr(), slot.numel(),
                                                   out.data_ptr(), self._stream()))
        return out

    def lower_bound_native(self, comm, q: torch.Tensor, fn=None):
        out, fb = self._u64(q.numel()), torch.zeros(1, dtype=torch.int64, device=self.device)
        api._check((fn or self.lib.rmi_shard_index_lower_bound)(self._h, comm, q.data_ptr(), q.numel(), out.data_ptr(),
                                                                fb.data_ptr(), self._stream()))
        return out, fb

    def upper_bound_native(self, comm, q: torch.Tensor):
        return self.lower_bound_native(comm, q, self.lib.rmi_shard_index_upper_bound)

    def last_stats(self) -> dict:
        st = _LookupStats()
        api._check(self.lib.rmi_shard_index_last_stats(self._h, C.byref(st)))
        return dict(phase_ms=dict(zip(LOOKUP_PHASES, (float(x) for x in st.phase_ms))),
                    queries_routed=int(st.queries_routed), queries_searched=int(st.queries_searched),
                    queries_kept=int(st.queries_kept))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.rmi_shard_index_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CudaShardEval:
    """One rank's side of evaluate_sharded on librmi_b200.so (rmi_shard_eval_*).  bounds / keys enqueue on the current
    torch stream of the data's device and return device tensors (int64 storage of the u64 words)."""

    def __init__(self, eng: CudaShardEngine, trained, ends_all: np.ndarray, world: int, rank: int):
        L = self.lib = api.load_library()
        L.rmi_shard_eval_create.argtypes = [C.POINTER(api._Result), C.c_void_p, C.POINTER(_Ends), C.c_int, C.c_int,
                                            C.POINTER(C.c_void_p)]
        L.rmi_shard_eval_destroy.argtypes = [C.c_void_p]
        L.rmi_shard_eval_partial_words.argtypes = [C.c_void_p]
        L.rmi_shard_eval_partial_words.restype = C.c_uint64
        L.rmi_shard_eval_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_shard_eval_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rmi_shard_eval_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                            C.POINTER(C.POINTER(api._Result))]
        L.rmi_shard_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.POINTER(api._Result))]
        self.device = eng.device
        self._ds = eng.ds             # the slab and the result are read at every evaluation: kept alive with it
        self._trained = trained
        self._spec = trained.models
        self.N = int(trained.branching_factor)
        self._h = C.c_void_p()
        api._check(L.rmi_shard_eval_create(api._result_ptr(trained), eng.ds._h, _ends_array(ends_all), world, rank,
                                           C.byref(self._h)))
        self.partial_words = int(L.rmi_shard_eval_partial_words(self._h))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream or None)

    def bounds(self) -> torch.Tensor:
        S = torch.empty(self.N + 1, dtype=torch.int64, device=self.device)
        api._check(self.lib.rmi_shard_eval_bounds(self._h, S.data_ptr(), self._stream()))
        return S

    def keys(self, S: torch.Tensor):
        part = torch.empty(2 * self.N, dtype=torch.int64, device=self.device)
        status = torch.zeros(1, dtype=torch.int32, device=self.device)
        api._check(self.lib.rmi_shard_eval_keys(self._h, S.data_ptr(), part.data_ptr(), status.data_ptr(), self._stream()))
        return part, status

    def finish(self, S: torch.Tensor, part: torch.Tensor, status: int, flags: int):
        res = C.POINTER(api._Result)()
        api._check(self.lib.rmi_shard_eval_finish(self._h, S.data_ptr(), part.data_ptr(), int(status), int(flags),
                                                  C.byref(res)))
        return api.result_from_pointer(res, self._spec)

    def evaluate(self, comm, flags: int):
        res = C.POINTER(api._Result)()
        api._check(self.lib.rmi_shard_evaluate(self._h, comm, int(flags), C.byref(res)))
        return api.result_from_pointer(res, self._spec)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.rmi_shard_eval_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardedRMIIndex:
    """A trained RMI served over range-partitioned keys: rank r holds the r-th slab (`data`, a ShardedTrainingData)
    and the whole model.  `trained` is any TrainedRMI of the whole key set: from train_sharded, from rmi_train of the
    whole keys, or loaded from an artefact (ShardedRMIIndex.load).  Constructing it gathers the ends of every slab once
    (cached on `data`, shared with train_sharded).

    predict(q) -> (pos, err): the model's prediction over the whole key set; local, no communication.
    lower_bound(q): exact global lower bounds (np.searchsorted(all_keys, q, "left"); 0 for NaN); collective: every
    rank calls it, with its own queries (0 is fine).  upper_bound(q): exact global upper bounds
    (np.searchsorted(all_keys, q, "right"); 0 for NaN), routed by <= (DESIGN §18); equal_range(q): lower_bound then
    upper_bound, two exchanges.  Under an NCCL group it is one library call (route, exchanges,
    search, gather on the stream); otherwise (gloo, native=False) the phases are driven here with all_to_all_single.
    Queries are a 1-D tensor on the data's device in its storage dtype (int64 for uint64 keys, int32, float64);
    results are int64 tensors (uint64 values) there.  The orchestration is engine-agnostic: the CPU tests plug in a
    numpy engine (`engine=`)."""

    def __init__(self, trained, data, group=None, engine=None):
        eng = engine if engine is not None else data.engine
        self.group = group if group is not None else getattr(data, "group", None)
        self.rank, self.world = _world(self.group)
        self.device = eng.device
        self.key_type = data.key_type
        self.index = eng.lookup_index(trained, gather_ends(data, eng, self.group), self.world, self.rank)

    @classmethod
    def load(cls, namespace: str, data, out_dir: str = ".", data_dir: str = "rmi_data", group=None,
             evaluate: bool = False) -> "ShardedRMIIndex":
        """load_rmi of a generated artefact, served over the slabs: train once, serve over shards.  evaluate=True
        measures the artefact's error bounds over the slabs first (evaluate_sharded, collective): a --no-errors
        artefact, or one whose keys have changed since it was generated, is then served with bounds that hold."""
        trained, cf = api.load_rmi(namespace, out_dir, data_dir)
        if cf is not None:
            raise api.RMIError("a --bounded artefact cannot be served over range-partitioned keys: its cache-fix spline "
                               "indexes the whole key array on one GPU")
        if trained.last_layer_max_l1s is None and not evaluate:
            raise api.RMIError("a --no-errors artefact holds no error bounds: load it with evaluate=True to measure them "
                               "over the slabs")
        want = (api.KEY_F64,) if trained.key_type == api.KEY_F64 else (api.KEY_U64, api.KEY_U32)
        if data.key_type not in want:
            raise api.RMIError(f"the artefact's lookup takes {'double' if trained.key_type == api.KEY_F64 else 'uint64_t'} "
                               f"keys, the data holds {np.dtype(_NP_OF_KEY[data.key_type])}")
        if evaluate:
            trained = evaluate_sharded(trained, data, group=group)
        return cls(trained, data, group)

    def _queries(self, q: torch.Tensor) -> torch.Tensor:
        want = _TORCH_OF_KEY[self.key_type]
        if not isinstance(q, torch.Tensor) or q.dtype != want or q.dim() != 1 or q.device != self.device:
            got = f"{q.dtype} on {q.device}" if isinstance(q, torch.Tensor) else type(q).__name__
            raise TypeError(f"queries must be a 1-D {want} tensor on {self.device}, got {got}")
        return q.contiguous()

    def predict(self, q: torch.Tensor):
        """(pos, err) per query over the whole key set."""
        return self.index.predict(self._queries(q))

    def lower_bound(self, q: torch.Tensor, return_fallbacks: bool = False, native: bool | None = None):
        """Exact global lower bounds of this rank's queries.  return_fallbacks: also the number of windows that
        missed among the queries THIS rank searched (the sum over ranks covers every query once)."""
        return self._bound(q, return_fallbacks, native, upper=False)

    def upper_bound(self, q: torch.Tensor, return_fallbacks: bool = False, native: bool | None = None):
        """Exact global upper bounds of this rank's queries (the number of keys <= q; 0 for NaN); return_fallbacks
        and native as for lower_bound."""
        return self._bound(q, return_fallbacks, native, upper=True)

    def equal_range(self, q: torch.Tensor, return_fallbacks: bool = False, native: bool | None = None):
        """(first, last): lower_bound(q) and upper_bound(q), one exchange each; return_fallbacks: also the sum of
        the two calls' counts."""
        first, fb_lo = self.lower_bound(q, True, native)
        last, fb_hi = self.upper_bound(q, True, native)
        return (first, last, fb_lo + fb_hi) if return_fallbacks else (first, last)

    def _bound(self, q: torch.Tensor, return_fallbacks: bool, native: bool | None, upper: bool):
        q = self._queries(q)
        comm = None
        if native is not False and isinstance(self.index, CudaShardIndex):
            comm = native_comm(self.group, self.device, single_rank_ok=native is True)
            if native is True and comm is None:
                raise api.RMIError("native=True needs an NCCL process group (or a single rank) and a loadable libnccl.so.2")
        if comm is not None:
            out, fb = (self.index.upper_bound_native if upper else self.index.lower_bound_native)(comm, q)
        elif upper:
            out, fb = self._phases(q, self.index.route_upper, self.index.search_upper)
        else:
            out, fb = self._lower_bound_phases(q)
        return (out, int(fb)) if return_fallbacks else out

    def _lower_bound_phases(self, q: torch.Tensor):
        return self._phases(q, self.index.route, self.index.search)

    def _phases(self, q: torch.Tensor, route, search):
        """route -> count exchange -> query exchange -> search -> answer exchange -> gather, the exchanges through
        torch.distributed.  search(received) -> (answers, fallbacks)."""
        idx, group = self.index, self.group
        send, slot, counts = route(q)
        if self.world <= 1:
            answers, fb = search(send)
            return idx.gather(slot, answers), fb
        # gloo cannot exchange device memory (one-GPU test boxes): stage through the host there
        stage = self.device.type == "cuda" and dist.get_backend(group) == "gloo"
        c_send = counts.cpu() if stage else counts
        c_recv = torch.empty_like(c_send)
        dist.all_to_all_single(c_recv, c_send, group=group)
        scount, rcount = c_send.tolist(), c_recv.tolist()      # the one host read of the counts
        recv = self._exchange(send, rcount, scount, stage)
        answers, fb = search(recv)
        returned = self._exchange(answers, scount, rcount, stage)
        return idx.gather(slot, returned), fb

    def _exchange(self, x: torch.Tensor, out_splits: list[int], in_splits: list[int], stage: bool) -> torch.Tensor:
        src = x.cpu() if stage else x
        out = torch.empty(sum(out_splits), dtype=x.dtype, device=src.device)
        dist.all_to_all_single(out, src, output_split_sizes=out_splits, input_split_sizes=in_splits, group=self.group)
        return out.to(self.device) if stage else out

    def close(self):
        if hasattr(self.index, "close"):
            self.index.close()


# ---- the cache-fix spline over the slabs (include/rmi_b200.h rmi_shard_cache_fix_*, DESIGN.md section 16) -----------

class _CacheFixScan(C.Structure):
    _fields_ = [("exit_pid", C.c_uint64), ("num_knots", C.c_uint64), ("reach", C.c_uint64), ("status", C.c_uint32),
                ("_pad", C.c_uint32)]


PID_END = (1 << 64) - 1            # RMI_SHARD_CACHE_FIX_PID_END: the last segment stays open to the end of the data
CACHE_FIX_HALO_TOO_SMALL = 1       # RMI_SHARD_CACHE_FIX_HALO_TOO_SMALL


class CudaShardCacheFix:
    """One rank's side of cache_fix_sharded on librmi_b200.so (rmi_shard_cache_fix_*), on the current torch stream of
    the data's device.  scan(entry) -> (exit pid, status, reach, knots to emit); emit() -> the knots as a (K, 2) int64
    tensor (uint64 key, offset) on the device."""

    def __init__(self, eng: CudaShardEngine, ends_all: np.ndarray, world: int, rank: int, line_size: int,
                 halo_keys: int):
        L = self.lib = api.load_library()
        L.rmi_shard_cache_fix_create.argtypes = [C.c_void_p, C.POINTER(_Ends), C.c_int, C.c_int, C.c_uint64, C.c_uint64,
                                                 C.c_void_p, C.POINTER(C.c_void_p)]
        L.rmi_shard_cache_fix_scan.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(_CacheFixScan)]
        L.rmi_shard_cache_fix_emit.argtypes = [C.c_void_p, C.c_void_p]
        L.rmi_shard_cache_fix_destroy.argtypes = [C.c_void_p]
        self.device = eng.device
        self._ds = eng.ds             # the slab and its halo are read at every scan: kept alive with it
        self.num_knots = 0
        self._h = C.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream or None
        api._check(L.rmi_shard_cache_fix_create(eng.ds._h, _ends_array(ends_all), world, rank, int(line_size),
                                                int(halo_keys), C.c_void_p(stream), C.byref(self._h)))

    def scan(self, entry: int):
        r = _CacheFixScan()
        api._check(self.lib.rmi_shard_cache_fix_scan(self._h, int(entry), C.byref(r)))
        self.num_knots = int(r.num_knots)
        return int(r.exit_pid), int(r.status), int(r.reach), int(r.num_knots)

    def emit(self) -> torch.Tensor:
        out = torch.empty((self.num_knots, 2), dtype=torch.int64, device=self.device)
        api._check(self.lib.rmi_shard_cache_fix_emit(self._h, out.data_ptr() if self.num_knots else None))
        return out

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.rmi_shard_cache_fix_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _gather_rows(row: list[int], world: int, group, dev, stage: bool) -> list[list[int]]:
    """Every rank's row of u64 words, in rank order (a tiny all-gather; through the host under gloo)."""
    t = torch.from_numpy(np.array(row, dtype=np.uint64).view(np.int64))
    if world <= 1:
        return [list(row)]
    t = t if stage else t.to(dev)
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t, group=group)
    return [[int(v) for v in o.cpu().numpy().view(np.uint64)] for o in out]


def cache_fix_sharded(data, line_size: int, group=None, root_only: bool = False, engine=None,
                      timings: dict | None = None):
    """api.cache_fix of the concatenated slabs (u64 keys), fitted where the keys live (DESIGN.md section 16).  Returns
    the (K, 2) uint64 knot array on every rank, or on rank 0 only with root_only (None elsewhere); collective.  Each
    rank also keeps its own knots on its device as ``data.cache_fix_knots = (line_size, (K_r, 2) int64 tensor)``: a
    sorted slab of the knot set.  Raises the reference's panics (RMIPanic) on every rank alike, and RMIError for keys
    that are not u64.

    Every rank scans its slab from an entry point and reports its exit, the first knot at or past the next slab; ranks
    whose entry is not their predecessor's exit scan again from it until every entry agrees (at most world - 1 more
    rounds), then emit their knots.  A chain that needs keys past the halo fetched behind the slabs grows the halo
    and starts again.  timings: filled with the rounds and the host times (s) of the scans, rounds, emit and gather."""
    import time
    eng = engine if engine is not None else data.engine
    group = group if group is not None else getattr(data, "group", None)
    rank, world = _world(group)
    dev = eng.device
    ends_all = gather_ends(data, eng, group)
    bases = [0]
    for n_local in ends_all[:, 3]:
        bases.append(bases[-1] + int(n_local))
    n_global = bases[-1]
    if world > 1 and getattr(data, "_halo_have", None) is None:
        cap = _min_halo_capacity(data, group, world, dev)
        moves = plan_halo(bases, [bases[g + 1] + cap - 1 for g in range(world)], n_global)
        data._halo_have = _exchange_halo(eng, moves, rank, group, dev)
    stage = world > 1 and dev.type == "cuda" and dist.get_backend(group) == "gloo"

    def sync():
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)

    t = {} if timings is None else timings
    cf = eng.cache_fixer(ends_all, world, rank, line_size, getattr(data, "_halo_have", 0) or 0)
    try:
        t0 = time.perf_counter()
        entry = 2 * bases[rank]                      # this rank's own first point
        exit_pid, status, reach, count = cf.scan(entry)
        t["first_scan_s"] = time.perf_counter() - t0
        rounds, t0 = 0, time.perf_counter()
        while True:
            table = _gather_rows([entry, exit_pid, status, reach, count], world, group, dev, stage)
            if any(row[2] & CACHE_FIX_HALO_TOO_SMALL for row in table):
                cf.close()
                return _cache_fix_with_larger_halo(data, line_size, group, root_only, engine, timings, table, bases)
            moved = False
            for r in range(1, world):
                if table[r][0] != table[r - 1][1]:
                    moved = True
                    if r == rank:
                        entry = table[r - 1][1]
                        exit_pid, status, reach, count = cf.scan(entry)
            if not moved:
                break
            rounds += 1
        t["join_rounds"] = rounds
        t["join_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        local = cf.emit()
        sync()
        t["emit_s"] = time.perf_counter() - t0
    finally:
        cf.close()
    data.cache_fix_knots = (int(line_size), local)
    t0 = time.perf_counter()
    counts = [row[4] for row in table]
    if world <= 1:
        knots = local.cpu()
    else:
        # equal-sized pieces for the collective: every rank's knots padded to the largest count
        send = torch.zeros((max(counts), 2), dtype=torch.int64, device="cpu" if stage else dev)
        send[: counts[rank]].copy_(local)
        if root_only:
            parts = [torch.empty_like(send) for _ in range(world)] if rank == 0 else None
            dist.gather(send, parts, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        else:
            parts = [torch.empty_like(send) for _ in range(world)]
            dist.all_gather(parts, send, group=group)
        knots = torch.cat([p[:c] for p, c in zip(parts, counts)]).cpu() if parts is not None else None
    t["gather_s"] = time.perf_counter() - t0
    if knots is None or (root_only and rank != 0):
        return None
    return knots.numpy().view(np.uint64).reshape(-1, 2)


def _cache_fix_with_larger_halo(data, line_size, group, root_only, engine, timings, table, bases):
    # A chain reaches past the halo.  Every rank saw the same table: grow every halo past the furthest walk and redo.
    if not hasattr(data, "grow_halo"):
        raise api.RMIError("the cache-fix spline reaches past the halo copied from the next ranks")
    need = max(row[3] - bases[r + 1] for r, row in enumerate(table) if row[2] & CACHE_FIX_HALO_TOO_SMALL)
    data.grow_halo(2 * max(need, data.halo_capacity) + 256)
    return cache_fix_sharded(data, line_size, group, root_only, None, timings)


def train_bounded_sharded(data, model_spec: str, num_leaves: int, line_size: int, flags: int = 0, group=None,
                          halo_capacity: int = 1 << 20):
    """api.train_bounded over range-partitioned keys: returns (TrainedRMI with num_data_rows = the keys of all slabs,
    knots), the pair api.train_bounded returns for the concatenated keys, on every rank; collective.  The spline is
    fitted by cache_fix_sharded, then train_sharded builds the RMI over every rank's slab of knot keys (a
    ShardedTrainingData with halo_capacity keys of room), so no knot table has to fit on one GPU.
    api.output_rmi(..., cache_fix_knots=knots, line_size=line_size) then writes the reference's `--bounded` artefact."""
    group = group if group is not None else getattr(data, "group", None)
    knots = cache_fix_sharded(data, line_size, group)
    _, local = data.cache_fix_knots
    kdata = ShardedTrainingData(local[:, 0].contiguous(), key_type=api.KEY_U64, halo_capacity=halo_capacity,
                                group=group)
    rmi = train_sharded(kdata, model_spec, num_leaves, flags, group)
    rmi.num_data_rows = int(gather_ends(data, data.engine, group)[:, 3].astype(np.uint64).sum())
    return rmi, knots


# ---- `--bounded` lookups over the slabs (include/rmi_b200.h rmi_shard_index_create_bounded, DESIGN.md section 17) -------

def knot_halo_width(trained) -> int:
    """h = 2 e_max + 2 knots on each side of a rank's knot slab, e_max the largest leaf error bound of the knot RMI
    (its last_layer_max_l1s: a loaded artefact holds no statistics).  DESIGN.md section 17 gives the bound."""
    errs = getattr(trained, "last_layer_max_l1s", None)
    if errs is None:
        raise api.RMIError("the knot RMI holds no error bounds (a --bounded artefact without errors cannot be served)")
    return 2 * int(np.max(np.asarray(errs, dtype=np.uint64))) + 2


def knot_owners(knot_keys: np.ndarray, ends_all: np.ndarray) -> np.ndarray:
    """The rank every knot key routes to by DESIGN.md section 14's rule: the last non-empty key slab whose first key is
    below it, or the first non-empty slab.  Pure function of the knot keys and gather_ends' table."""
    nonempty = np.flatnonzero(ends_all[:, 3].astype(np.uint64) > 0)
    firsts = ends_all[nonempty, 0].astype(np.uint64)
    below = np.searchsorted(firsts, np.asarray(knot_keys, dtype=np.uint64), "left")
    return nonempty[np.maximum(below.astype(np.int64) - 1, 0)]


def plan_knot_halo(counts: list[int], rank: int, h: int) -> tuple[list[tuple[int, int, int, int]], list[tuple[int, int, int, int]]]:
    """Where rank's knot halo comes from, given every rank's knot count and the halo width h.  Rank p publishes its
    first and its last min(h, counts[p]) knots (its head and tail); the halo is global knots [max(a0 - h, 0), a0)
    before the slab [a0, a1) and [a1, min(a1 + h, K)) after it.  Returns (before, after): pieces (src rank, side, offset,
    count) in global order, side 0 = src's head, 1 = its tail, offset into that side.  Every knot within h of a slab
    lies in its owner's head or tail, so the pieces cover both ranges, across any number of ranks with few or no knots."""
    bases = [0]
    for c in counts:
        bases.append(bases[-1] + int(c))
    K, a0, a1 = bases[-1], bases[rank], bases[rank + 1]
    before, after = [], []
    for p in range(len(counts)):
        lo, hi, w = bases[p], bases[p + 1], min(h, int(counts[p]))
        if p < rank:                                   # from p's tail: global [hi - w, hi)
            g0, g1 = max(hi - w, a0 - h, 0), min(hi, a0)
            if g1 > g0:
                before.append((p, 1, g0 - (hi - w), g1 - g0))
        elif p > rank:                                 # from p's head: global [lo, lo + w)
            g0, g1 = max(lo, a1), min(lo + w, a1 + h, K)
            if g1 > g0:
                after.append((p, 0, g0 - lo, g1 - g0))
    return before, after


def _all_gather_u64(row: np.ndarray, world: int, group, dev, stage: bool) -> np.ndarray:
    """Every rank's equal-length row of u64 words as a (world, len) array (a small all-gather; through the host under
    gloo)."""
    t = torch.from_numpy(np.ascontiguousarray(row, dtype=np.uint64).view(np.int64))
    if world <= 1:
        return np.ascontiguousarray(row, dtype=np.uint64)[None, :]
    t = t if stage else t.to(dev)
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t, group=group)
    return torch.stack(out).cpu().numpy().view(np.uint64)


def _route_local_knots(local: np.ndarray, ends_all: np.ndarray, world: int, rank: int, group, dev, stage: bool):
    """From the knot slabs cache_fix_sharded leaves (partitioned by point index), every rank's knot slab by the routing
    rule.  The knots that route elsewhere (a few at the cuts: the minus and key points of a slab's first key, and the
    final point when a slab is one repeated key) travel in one all-gather, padded to the most any rank sends, after one
    of every rank's (staying, moving) counts.  Returns (this rank's slab, every rank's knot count)."""
    dest = knot_owners(local[:, 0], ends_all) if len(local) else np.zeros(0, dtype=np.int64)
    stay, moving, mdest = local[dest == rank], local[dest != rank], dest[dest != rank]
    sizes = _all_gather_u64(np.array([len(stay), len(moving)], dtype=np.uint64), world, group, dev, stage)
    counts = [int(x) for x in sizes[:, 0]]
    width = int(sizes[:, 1].max())
    incoming = []
    if width:
        row = np.zeros((width, 3), dtype=np.uint64)
        row[: len(moving), :2] = moving
        row[: len(moving), 2] = mdest
        table = _all_gather_u64(row.reshape(-1), world, group, dev, stage).reshape(world, width, 3)
        for p in range(world):
            moved = table[p, : int(sizes[p, 1])]
            for d in moved[:, 2]:
                counts[int(d)] += 1
            incoming.append(moved[moved[:, 2] == rank, :2])
    slab = np.concatenate([stay] + incoming) if incoming else stay
    slab = slab[np.argsort(slab[:, 0], kind="stable")]
    return np.ascontiguousarray(slab, dtype=np.uint64).reshape(-1, 2), counts


def _assemble_halo(slab: np.ndarray, counts: list[int], h: int, world: int, rank: int, group, dev, stage: bool):
    """This rank's knot slab with its halo (plan_knot_halo) from one all-gather of every rank's head and tail of h
    knots.  Returns (knots, halo_before)."""
    w = min(h, len(slab))
    row = np.zeros(4 * h, dtype=np.uint64)
    row[: 2 * w] = slab[:w].reshape(-1)
    row[2 * h: 2 * h + 2 * w] = slab[len(slab) - w:].reshape(-1)
    table = _all_gather_u64(row, world, group, dev, stage)
    before, after = plan_knot_halo(counts, rank, h)

    def piece(src, side, off, cnt):
        return table[src, 2 * h * side:].reshape(-1, 2)[off: off + cnt]

    parts = [piece(*x) for x in before] + [slab] + [piece(*x) for x in after]
    return np.ascontiguousarray(np.concatenate(parts), dtype=np.uint64).reshape(-1, 2), sum(x[3] for x in before)


class CudaShardBoundedIndex(CudaShardIndex):
    """One rank's side of ShardedBoundedRMIIndex on librmi_b200.so (rmi_shard_index_create_bounded): the route, search
    and gather of CudaShardIndex, and the collective predict (predict_route / predict_search, or predict_native)."""

    def __init__(self, eng: CudaShardEngine, trained, knots: np.ndarray, halo_before: int, knot_counts: list[int],
                 line_size: int, ends_all: np.ndarray, world: int, rank: int):
        L = self._bind(eng, trained, world)
        L.rmi_shard_index_create_bounded.argtypes = [C.POINTER(api._Result), C.c_void_p, C.c_uint64, C.c_uint64,
                                                     C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(_Ends), C.c_int,
                                                     C.c_int, C.POINTER(C.c_void_p)]
        L.rmi_shard_index_predict_route.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p]
        L.rmi_shard_index_predict_search.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        L.rmi_shard_index_predict_collective.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                                         C.c_void_p, C.c_void_p]
        self.line_size = int(line_size)
        k = np.ascontiguousarray(knots, dtype=np.uint64).reshape(-1, 2)
        kc = np.ascontiguousarray(knot_counts, dtype=np.uint64)
        api._check(L.rmi_shard_index_create_bounded(
            api._result_ptr(trained), k.ctypes.data_as(C.c_void_p), k.shape[0], int(halo_before),
            kc.ctypes.data_as(C.c_void_p), self.line_size, eng.ds._h, _ends_array(ends_all), world, rank,
            C.byref(self._h)))

    def predict_route(self, q: torch.Tensor):
        send, slot, counts = torch.empty_like(q), self._u64(q.numel()), self._u64(self.world)
        api._check(self.lib.rmi_shard_index_predict_route(self._h, q.data_ptr(), q.numel(), send.data_ptr(),
                                                          slot.data_ptr(), counts.data_ptr(), self._stream()))
        return send, slot, counts

    def predict_search(self, recv: torch.Tensor):
        pos = self._u64(recv.numel())
        api._check(self.lib.rmi_shard_index_predict_search(self._h, recv.data_ptr(), recv.numel(), pos.data_ptr(),
                                                           self._stream()))
        return pos, 0

    def predict_native(self, comm, q: torch.Tensor):
        pos, err = self._u64(q.numel()), self._u64(q.numel())
        api._check(self.lib.rmi_shard_index_predict_collective(self._h, comm, q.data_ptr(), q.numel(), pos.data_ptr(),
                                                               err.data_ptr(), self._stream()))
        return pos, err


class ShardedBoundedRMIIndex(ShardedRMIIndex):
    """A `--bounded` RMI served over range-partitioned uint64 keys (DESIGN.md section 17).  `trained` is the RMI over
    the cache-fix spline's knots (from train_bounded_sharded, api.train_bounded of the whole keys, or an artefact:
    ShardedBoundedRMIIndex.load); `data` a ShardedTrainingData of uint64 slabs; `knots` the whole (K, 2) knot array
    (the same on every rank), or None to take each rank's knots from data.cache_fix_knots, which cache_fix_sharded
    leaves on its device.  No rank holds every knot: rank r keeps the knots whose key routes to it and a halo of
    h = 2 e_max + 2 knots on each side (knot_halo_width), assembled once here from one small all-gather.

    lower_bound(q): collective, exact (np.searchsorted(all_keys, q, "left")), routed by key as ShardedRMIIndex's.
    predict(q) -> (pos, err): collective (unlike ShardedRMIIndex.predict), routed by knot index; bit for bit the
    one-GPU BoundedRMIIndex(trained, all_knots, line_size, all_keys).predict, err = line_size.  return_fallbacks and
    native= behave as on ShardedRMIIndex.  Constructing it is collective."""

    def __init__(self, trained, knots, line_size: int, data, group=None, engine=None):
        eng = engine if engine is not None else data.engine
        self.group = group if group is not None else getattr(data, "group", None)
        self.rank, self.world = _world(self.group)
        self.device = eng.device
        self.key_type = data.key_type
        self.line_size = int(line_size)
        if data.key_type != api.KEY_U64:
            raise api.RMIError("Can only construct a bounded RMI on u64 data")
        h = knot_halo_width(trained)
        ends_all = self.ends_all = gather_ends(data, eng, self.group)
        if knots is not None:
            k = np.ascontiguousarray(knots, dtype=np.uint64).reshape(-1, 2)
            counts = np.bincount(knot_owners(k[:, 0], ends_all), minlength=self.world).tolist()
            a0 = sum(counts[: self.rank])
            a1 = a0 + counts[self.rank]
            lo = max(a0 - h, 0)
            ext, halo_before = k[lo: min(a1 + h, k.shape[0])], a0 - lo
        else:
            line, local = getattr(data, "cache_fix_knots", (None, None))
            if local is None:
                raise api.RMIError("knots=None needs the knot slabs cache_fix_sharded leaves on the data")
            if int(line) != self.line_size:
                raise api.RMIError(f"the knot slabs on the data are for line size {line}, not {self.line_size}")
            stage = self.world > 1 and self.device.type == "cuda" and dist.get_backend(self.group) == "gloo"
            local = local.cpu().numpy().view(np.uint64).reshape(-1, 2)
            slab, counts = _route_local_knots(local, ends_all, self.world, self.rank, self.group, self.device, stage)
            ext, halo_before = _assemble_halo(slab, counts, h, self.world, self.rank, self.group, self.device, stage)
        self.knot_counts = [int(c) for c in counts]
        self.index = eng.bounded_lookup_index(trained, ext, int(halo_before), self.knot_counts, self.line_size,
                                              ends_all, self.world, self.rank)

    @classmethod
    def load(cls, namespace: str, data, out_dir: str = ".", data_dir: str = "rmi_data",
             group=None) -> "ShardedBoundedRMIIndex":
        """load_rmi of a generated `--bounded` artefact, served over the slabs with its whole knot array."""
        trained, cf = api.load_rmi(namespace, out_dir, data_dir)
        if cf is None:
            raise api.RMIError("not a --bounded artefact: serve it with ShardedRMIIndex.load")
        if trained.last_layer_max_l1s is None:
            raise api.RMIError("a --bounded artefact without errors cannot be served")
        if data.key_type != api.KEY_U64:
            raise api.RMIError(f"the artefact's lookup takes uint64_t keys, the data holds "
                               f"{np.dtype(_NP_OF_KEY[data.key_type])}")
        return cls(trained, cf[1], cf[0], data, group)

    def predict(self, q: torch.Tensor, native: bool | None = None):
        """(pos, err) per query: the one-GPU bounded index's, bit for bit; collective (every rank calls it)."""
        q = self._queries(q)
        comm = None
        if native is not False and isinstance(self.index, CudaShardBoundedIndex):
            comm = native_comm(self.group, self.device, single_rank_ok=native is True)
            if native is True and comm is None:
                raise api.RMIError("native=True needs an NCCL process group (or a single rank) and a loadable libnccl.so.2")
        if comm is not None:
            return self.index.predict_native(comm, q)
        pos, _ = self._phases(q, self.index.predict_route, self.index.predict_search)
        return pos, torch.full_like(pos, self.line_size)
