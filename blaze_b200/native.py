"""ctypes binding of the C ABI (include/blaze_b200.h) — plays the role of the reference's Rust host
(`ExecutionPlan::execute` shims, INTEGRATION.md) in tests, smoke and bench.

There is NO CPU fallback here: if `libblaze_b200.so` is missing this module raises at import, and if
no CUDA device is visible `NativeOp(...)` raises `NativeError(B200Q_ERR_NO_DEVICE)`.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libblaze_b200.so")

OK, ERR_INVALID_PLAN, ERR_UNSUPPORTED, ERR_CUDA, ERR_STATE, ERR_EXECUTION, ERR_NO_DEVICE, ERR_INVALID_ARG = range(8)
PLAN_NODE, TASK_DEFINITION = 0, 1
ARROW_DEVICE_CUDA = 2


class NativeError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"[b200q status {code}] {msg}")
        self.code = code
        self.msg = msg


class ArrowSchema(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
    ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchema))), ("dictionary", C.POINTER(ArrowSchema)),
    ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArray(C.Structure):
    pass


ArrowArray._fields_ = [
    ("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
    ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)), ("children", C.POINTER(C.POINTER(ArrowArray))),
    ("dictionary", C.POINTER(ArrowArray)), ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowDeviceArray(C.Structure):
    _fields_ = [("array", ArrowArray), ("device_id", C.c_int64), ("device_type", C.c_int32),
                ("sync_event", C.c_void_p), ("reserved", C.c_int64 * 3)]


class Conf(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("batch_size", C.c_int32), ("suggested_batch_mem_size", C.c_int64),
                ("partial_agg_skipping_enable", C.c_int32), ("partial_agg_skipping_ratio", C.c_double),
                ("partial_agg_skipping_min_rows", C.c_int64), ("staging_rows", C.c_int64),
                ("agg_initial_groups", C.c_int64), ("max_launch_rows", C.c_int64),
                ("partial_state_columnar", C.c_int32), ("force_generic_kernels", C.c_int32), ("agg_dense_keys", C.c_int32), ("agg_hot_key_cache", C.c_int32),
                ("agg_max_table_bytes", C.c_int64), ("shuffle_output_on_device", C.c_int32)]


class ShuffleChunk(C.Structure):
    _fields_ = [("data", C.c_void_p), ("on_device", C.c_int32), ("num_partitions", C.c_int32), ("rows", C.c_int64),
                ("part_off", C.POINTER(C.c_uint64)), ("part_rows", C.POINTER(C.c_uint64))]


class Metrics(C.Structure):
    _fields_ = [("struct_size", C.c_uint32)] + [(n, C.c_int64) for n in (
        "input_rows", "input_batches", "output_rows", "output_batches", "elapsed_compute_ns", "gpu_kernel_launches",
        "h2d_bytes", "d2h_bytes", "num_groups", "table_capacity_slots", "table_grow_count", "fast_path_launches",
        "hot_kernel_ns", "hot_kernel_rows", "hot_kernel_launches")]


# every symbol include/blaze_b200.h declares (tests/test_capi_symbols.py checks the .so exports them all)
SYMBOLS = ["b200q_version", "b200q_build_info", "b200q_last_error", "b200q_device_count", "b200q_conf_init",
           "b200q_plan_explain", "b200q_op_create", "b200q_op_input_schema", "b200q_op_output_schema", "b200q_op_push",
           "b200q_op_push_device", "b200q_op_finish", "b200q_op_pull", "b200q_op_pull_device", "b200q_op_sync",
           "b200q_op_metrics", "b200q_op_destroy", "b200q_murmur3_partition",
           "b200q_set_file_reader", "b200q_parquet_explain", "b200q_snappy_uncompress", "b200q_op_attach_build", "b200q_op_attach_right", "b200q_op_shuffle_chunk_count", "b200q_op_shuffle_chunk", "b200q_lz4_frame_compress",
           "b200q_lz4_frame_decompress", "b200q_op_push_ipc", "b200q_set_scalar_subquery_resolver",
           "b200q_exchange_unique_id", "b200q_exchange_create", "b200q_exchange_shuffle", "b200q_exchange_kernel_launches",
           "b200q_exchange_destroy"]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback for the hot path)")
    lib = C.CDLL(LIB_PATH)
    lib.b200q_version.restype = C.c_int32
    lib.b200q_build_info.restype = C.c_char_p
    lib.b200q_last_error.restype = C.c_char_p
    lib.b200q_device_count.restype = C.c_int32
    lib.b200q_conf_init.argtypes = [C.POINTER(Conf)]
    lib.b200q_plan_explain.argtypes = [C.c_char_p, C.c_size_t, C.c_int32, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.b200q_op_create.argtypes = [C.c_char_p, C.c_size_t, C.c_int32, C.c_void_p, C.POINTER(Conf), C.c_int32, C.POINTER(C.c_void_p)]
    for n in ("b200q_op_input_schema", "b200q_op_output_schema"):
        getattr(lib, n).argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_op_push.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_op_push_device.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_op_finish.argtypes = [C.c_void_p]
    lib.b200q_op_sync.argtypes = [C.c_void_p]
    lib.b200q_op_pull.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
    lib.b200q_op_pull_device.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
    lib.b200q_op_metrics.argtypes = [C.c_void_p, C.POINTER(Metrics)]
    lib.b200q_op_destroy.argtypes = [C.c_void_p]
    lib.b200q_op_destroy.restype = None
    lib.b200q_murmur3_partition.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.b200q_set_file_reader.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_parquet_explain.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.b200q_snappy_uncompress.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.b200q_op_attach_build.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_op_attach_right.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_op_shuffle_chunk_count.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    lib.b200q_op_shuffle_chunk.argtypes = [C.c_void_p, C.c_int64, C.POINTER(ShuffleChunk)]
    lib.b200q_lz4_frame_compress.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.b200q_lz4_frame_decompress.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.b200q_op_push_ipc.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    lib.b200q_set_scalar_subquery_resolver.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200q_exchange_unique_id.argtypes = [C.c_void_p]
    lib.b200q_exchange_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    lib.b200q_exchange_shuffle.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.b200q_exchange_kernel_launches.argtypes = [C.c_void_p]
    lib.b200q_exchange_kernel_launches.restype = C.c_int64
    lib.b200q_exchange_destroy.argtypes = [C.c_void_p]
    lib.b200q_exchange_destroy.restype = None
    return lib


lib = _load()


def parquet_explain(footer: bytes) -> str:
    """host-only: the library's view of a parquet FileMetaData footer"""
    need = C.c_size_t(0)
    check(lib.b200q_parquet_explain(footer, len(footer), None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib.b200q_parquet_explain(footer, len(footer), buf, need.value, C.byref(need)))
    return buf.value.decode()


def snappy_uncompress(data: bytes, capacity: int) -> bytes:
    out = C.create_string_buffer(max(1, capacity))
    n = C.c_size_t(0)
    check(lib.b200q_snappy_uncompress(data, len(data), out, capacity, C.byref(n)))
    return out.raw[: n.value]


def lz4_frame_compress(data: bytes) -> bytes:
    """the library's own LZ4 frame encoder (host only): the compression blocks of the shuffle files"""
    need = C.c_size_t(0)
    cap = len(data) + len(data) // 255 + 64
    buf = C.create_string_buffer(cap)
    check(lib.b200q_lz4_frame_compress(data, len(data), buf, cap, C.byref(need)))
    return buf.raw[: need.value]


def lz4_frame_decompress(data: bytes) -> bytes:
    """the library's own LZ4 frame decoder (host only): the compression blocks the reduce side reads"""
    need = C.c_size_t(0)
    st = lib.b200q_lz4_frame_decompress(data, len(data), None, 0, C.byref(need))
    if st != ERR_INVALID_ARG or "needs" not in last_error():
        check(st)
    buf = C.create_string_buffer(max(1, need.value))
    check(lib.b200q_lz4_frame_decompress(data, len(data), buf, need.value, C.byref(need)))
    return buf.raw[: need.value]


_BYTES_SINK = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_size_t)
_SUBQUERY_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.POINTER(C.c_uint8), C.c_size_t, C.c_void_p, C.c_void_p)
_resolver_keepalive = None


def set_scalar_subquery_resolver(fn) -> None:
    """Register `fn(serialized: bytes) -> bytes | None` as the process-wide scalar-subquery resolver
    (b200q_set_scalar_subquery_resolver): op create calls it once per BloomFilterMightContain whose filter is a ScalarSubquery.
    None removes it.  An exception raised by `fn` fails the create with ERR_EXECUTION."""
    global _resolver_keepalive
    if fn is None:
        check(lib.b200q_set_scalar_subquery_resolver(None, None))
        _resolver_keepalive = None
        return

    def trampoline(_ctx, serialized, n, put, sink):
        try:
            v = fn(C.string_at(serialized, n) if n else b"")
        except Exception:
            return 1
        if v is not None:
            v = bytes(v)
            _BYTES_SINK(put)(sink, C.cast(C.c_char_p(v), C.c_void_p), len(v))
        return 0

    cb = _SUBQUERY_FN(trampoline)
    check(lib.b200q_set_scalar_subquery_resolver(C.cast(cb, C.c_void_p), None))
    _resolver_keepalive = cb                    # the library holds the pointer: keep the ctypes thunk alive


def last_error() -> str:
    return (lib.b200q_last_error() or b"").decode("utf-8", "replace")


def check(status: int):
    if status != OK:
        raise NativeError(status, last_error())


def device_count() -> int:
    return int(lib.b200q_device_count())


def default_conf(**overrides) -> Conf:
    c = Conf()
    check(lib.b200q_conf_init(C.byref(c)))
    for k, v in overrides.items():
        if not hasattr(c, k):
            raise AttributeError(f"b200q_conf has no field {k!r}")
        setattr(c, k, v)
    return c


def plan_explain(plan_bytes: bytes, kind: int = PLAN_NODE) -> str:
    need = C.c_size_t(0)
    check(lib.b200q_plan_explain(plan_bytes, len(plan_bytes), kind, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value + 1)
    check(lib.b200q_plan_explain(plan_bytes, len(plan_bytes), kind, buf, len(buf), C.byref(need)))
    return buf.value.decode()


_RELEASE_CB = C.CFUNCTYPE(None, C.POINTER(ArrowArray))


class DeviceBatch:
    """A struct-typed ArrowDeviceArray over device pointers (torch tensors or raw addresses).

    columns: list of (values_ptr, validity_ptr_or_0, length) for fixed-width columns, and
    (data_ptr, validity_ptr_or_0, length, offsets_ptr) for Utf8 / Binary columns (int32 Arrow offsets).
    `keepalive` objects (the tensors) are held until the library calls release.
    """
    _live = {}

    def __init__(self, columns, num_rows: int, device: int, keepalive=()):
        self.n = len(columns)
        self.keepalive = list(keepalive)
        self.children = (ArrowArray * self.n)()
        self.child_ptrs = (C.POINTER(ArrowArray) * self.n)()
        self.buffers = []
        for i, col in enumerate(columns):
            vptr, nptr, ln = col[:3]
            b = (C.c_void_p * 3)(nptr or None, col[3], vptr) if len(col) == 4 else (C.c_void_p * 2)(nptr or None, vptr)
            self.buffers.append(b)
            c = self.children[i]
            c.length, c.null_count, c.offset, c.n_buffers, c.n_children = ln, (-1 if nptr else 0), 0, len(b), 0
            c.buffers = C.cast(b, C.POINTER(C.c_void_p))
            c.release = C.cast(_noop_release, C.c_void_p)
            self.child_ptrs[i] = C.pointer(c)
        self.top_buffers = (C.c_void_p * 1)(None)
        self.dev = ArrowDeviceArray()
        a = self.dev.array
        a.length, a.null_count, a.offset, a.n_buffers, a.n_children = num_rows, 0, 0, 1, self.n
        a.buffers = C.cast(self.top_buffers, C.POINTER(C.c_void_p))
        a.children = C.cast(self.child_ptrs, C.POINTER(C.POINTER(ArrowArray)))
        self._id = id(self)
        a.private_data = self._id
        a.release = C.cast(_device_release, C.c_void_p)
        self.dev.device_id = device
        self.dev.device_type = ARROW_DEVICE_CUDA
        DeviceBatch._live[self._id] = self        # released by the library through _device_release


@_RELEASE_CB
def _noop_release(p):
    p.contents.release = None


@_RELEASE_CB
def _device_release(p):
    DeviceBatch._live.pop(p.contents.private_data, None)
    p.contents.release = None


class NativeOp:
    """One operator pipeline handle (b200q_op)."""

    def __init__(self, plan_bytes: bytes, conf: Optional[Conf] = None, device: int = 0, kind: int = PLAN_NODE):
        self._h = C.c_void_p()
        conf = conf or default_conf()
        check(lib.b200q_op_create(plan_bytes, len(plan_bytes), kind, None, C.byref(conf), device, C.byref(self._h)))
        self.device = device

    # -- schemas
    def _schema(self, fn):
        import pyarrow as pa
        s = ArrowSchema()
        check(fn(self._h, C.addressof(s)))
        return pa.Schema._import_from_c(C.addressof(s))

    def input_schema(self):
        return self._schema(lib.b200q_op_input_schema)

    def output_schema(self):
        return self._schema(lib.b200q_op_output_schema)

    # -- data
    def push(self, rb):
        """rb: pyarrow.RecordBatch in host memory (ownership of the exported struct moves to the library)."""
        a = ArrowArray()
        s = ArrowSchema()
        rb._export_to_c(C.addressof(a), C.addressof(s))
        try:
            check(lib.b200q_op_push(self._h, C.addressof(a)))
        finally:
            import pyarrow as pa
            pa.Schema._import_from_c(C.addressof(s))     # releases the exported schema

    def push_ipc(self, data: bytes):
        """IpcReaderExec leaves: the bytes of one BlockObject (`u32 LE length ‖ LZ4 frame` blocks)"""
        check(lib.b200q_op_push_ipc(self._h, data, len(data)))

    def push_device(self, batch: DeviceBatch):
        check(lib.b200q_op_push_device(self._h, C.addressof(batch.dev)))

    def push_device_array(self, d: ArrowDeviceArray):
        """an ArrowDeviceArray produced by the library itself (pull_device / Exchange.shuffle); ownership moves to the op"""
        check(lib.b200q_op_push_device(self._h, C.addressof(d)))

    def finish(self):
        check(lib.b200q_op_finish(self._h))

    def sync(self):
        check(lib.b200q_op_sync(self._h))

    def pull(self):
        import pyarrow as pa
        a = ArrowArray()
        has = C.c_int32(0)
        check(lib.b200q_op_pull(self._h, C.addressof(a), C.byref(has)))
        if not has.value:
            return None
        s = ArrowSchema()
        check(lib.b200q_op_output_schema(self._h, C.addressof(s)))
        return pa.RecordBatch._import_from_c(C.addressof(a), C.addressof(s))

    def pull_all(self) -> List:
        out = []
        while True:
            b = self.pull()
            if b is None:
                return out
            out.append(b)

    def pull_device(self):
        """-> (ArrowDeviceArray struct, keep it alive; call release_device() when done) or None"""
        d = ArrowDeviceArray()
        has = C.c_int32(0)
        check(lib.b200q_op_pull_device(self._h, C.addressof(d), C.byref(has)))
        return d if has.value else None

    def attach_build(self, build_op: "NativeOp"):
        """join ops: use the finished map side held by `build_op` (a BroadcastJoinBuildHashMapExecNode op)"""
        check(lib.b200q_op_attach_build(self._h, build_op._h))

    def attach_right(self, right_op: "NativeOp"):
        """sort-merge join ops: take the queued output of `right_op` (finished, not pulled) as the join's right side"""
        check(lib.b200q_op_attach_right(self._h, right_op._h))

    def shuffle_chunks(self) -> List[dict]:
        """ShuffleWriterExec plans, after finish(): [{rows, part_off, part_rows, data (bytes, host) | data_ptr (device)}]"""
        n = C.c_int64(0)
        check(lib.b200q_op_shuffle_chunk_count(self._h, C.byref(n)))
        out = []
        for i in range(n.value):
            ch = ShuffleChunk()
            check(lib.b200q_op_shuffle_chunk(self._h, i, C.byref(ch)))
            P = ch.num_partitions
            off = [int(ch.part_off[j]) for j in range(P + 1)]
            d = {"rows": int(ch.rows), "part_off": off, "part_rows": [int(ch.part_rows[j]) for j in range(P)], "on_device": bool(ch.on_device)}
            if ch.on_device:
                d["data_ptr"] = int(ch.data or 0)
            else:
                d["data"] = C.string_at(ch.data, off[P]) if off[P] else b""
            out.append(d)
        return out

    def metrics(self) -> dict:
        m = Metrics()
        m.struct_size = C.sizeof(Metrics)
        check(lib.b200q_op_metrics(self._h, C.byref(m)))
        return {n: getattr(m, n) for n, _ in Metrics._fields_ if n != "struct_size"}

    def close(self):
        if self._h:
            lib.b200q_op_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def release_device_array(d: ArrowDeviceArray):
    if d.array.release:
        C.CFUNCTYPE(None, C.c_void_p)(d.array.release)(C.addressof(d.array))


def exchange_unique_id() -> bytes:
    """rank 0: the 128-byte ncclUniqueId every rank passes to Exchange(...); distribute it over the host's control plane"""
    buf = C.create_string_buffer(128)
    check(lib.b200q_exchange_unique_id(buf))
    return buf.raw


class Exchange:
    """b200q_exchange: murmur3(seed 42) pmod world repartitioning of device batches over NCCL (collective calls)."""

    def __init__(self, unique_id: bytes, rank: int, world: int, device: int):
        self._h = C.c_void_p()
        self.rank, self.world, self.device = rank, world, device
        check(lib.b200q_exchange_create(unique_id, rank, world, device, C.byref(self._h)))

    def shuffle(self, schema, dev_array: ArrowDeviceArray, n_key_cols: int) -> ArrowDeviceArray:
        """schema: pyarrow.Schema of the columns; dev_array is consumed; returns the rows this rank owns (release_device_array when done)"""
        s = ArrowSchema()
        schema._export_to_c(C.addressof(s))
        out = ArrowDeviceArray()
        try:
            check(lib.b200q_exchange_shuffle(self._h, C.addressof(s), C.addressof(dev_array), n_key_cols, C.addressof(out)))
        finally:
            import pyarrow as pa
            pa.Schema._import_from_c(C.addressof(s))
        return out

    def kernel_launches(self) -> int:
        return int(lib.b200q_exchange_kernel_launches(self._h))

    def close(self):
        if self._h:
            lib.b200q_exchange_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
