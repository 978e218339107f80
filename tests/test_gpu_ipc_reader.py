"""IpcReaderExec on the GPU through the C ABI: shuffle blocks (`u32 LE length ‖ LZ4 frame`, batch_serde records) decoded into device
batches, against oracle/shuffle_oracle.py::read_partition of the same bytes.  Every value is compared bit for bit (NaN payloads and
-0.0 included): fixed-width values as their little-endian bytes, Booleans and Binary / Utf8 values as such, NULLs by position."""
import decimal
import struct

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from blaze_b200.types import Field, Schema
from oracle import blaze_oracle as O
from oracle import shuffle_oracle as S
from helpers import *

pytestmark = pytest.mark.gpu

FIXED = {"i8": (T.int8, pa.int8()), "i16": (T.int16, pa.int16()), "i32": (T.int32, pa.int32()), "i64": (T.int64, pa.int64()),
         "f32": (T.float32, pa.float32()), "f64": (T.float64, pa.float64()), "date": (T.date32, pa.date32()),
         "ts": (T.timestamp_us, pa.timestamp("us")), "dec": (T.decimal128(38, 3), pa.decimal128(38, 3))}
ALL = list(FIXED) + ["bool", "bin", "utf8"]


def _array(rng, name, n, null_mode):
    """values of every bit pattern the type allows (NaN payloads, -0.0, ±inf, decimal at ±(10^38 - 1)); NULL slots hold 0"""
    mask = rng.random(n) < 0.1 if null_mode == "some" else np.zeros(n, bool)
    if name in ("bin", "utf8"):
        lens = rng.integers(0, 90, n)
        vals = [None if m else bytes(rng.integers(0, 256, int(ln), dtype=np.uint8)) for m, ln in zip(mask, lens)]
        return pa.array(vals, pa.binary())
    if name == "bool":
        return pa.array(rng.random(n) < 0.5, pa.bool_(), mask=mask if mask.any() else None)
    dt, pt = FIXED[name]
    if name == "dec":
        edge = [10**38 - 1, -(10**38 - 1), 0, 1, -1]
        ints = [edge[i % 5] if i % 7 == 0 else int(rng.integers(-10**18, 10**18)) * 10**int(rng.integers(0, 20)) for i in range(n)]
        raw = b"".join((0 if m else v).to_bytes(16, "little", signed=True) for v, m in zip(ints, mask))
        validity = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if mask.any() else None
        return pa.Array.from_buffers(pt, n, [validity, pa.py_buffer(raw)], null_count=int(mask.sum()))
    if name in ("f32", "f64"):
        w = 4 if name == "f32" else 8
        bits = rng.integers(0, 2**(8 * w) - 1, n, dtype=np.uint64 if w == 8 else np.uint32, endpoint=True)
        vals = bits.view(np.float64 if w == 8 else np.float32)
        special = np.array([np.nan, -0.0, np.inf, -np.inf, 0.0], vals.dtype)
        vals[::3] = special[np.arange(len(vals[::3])) % 5]
        vals = np.where(mask, 0, vals).astype(vals.dtype)
        return pa.array(vals, pt, mask=mask if mask.any() else None)
    info = np.iinfo({"i8": np.int8, "i16": np.int16, "i32": np.int32, "date": np.int32}.get(name, np.int64))
    vals = np.where(mask, 0, rng.integers(info.min, info.max, n, endpoint=True)).astype(info.dtype)
    return pa.array(vals, pt, mask=mask if mask.any() else None)


def _wire_schema(names, nullable=True):
    """the schema records are written with (Utf8 has Binary's wire form) and the one the plan reads them as"""
    types = {**{k: v[0] for k, v in FIXED.items()}, "bool": T.bool_, "bin": T.binary, "utf8": T.binary}
    wire = Schema([Field(n, types[n], nullable) for n in names])
    read = Schema([Field(n, T.utf8 if n == "utf8" else types[n], nullable) for n in names])
    return wire, read


def _records(rng, names, sizes, null_mode):
    """batch_serde bytes of one record per entry of `sizes`, as the oracle's write_batch writes them"""
    out = []
    for n in sizes:
        arrays = [_array(rng, nm, n, null_mode) for nm in names]
        if any(nm == "utf8" for nm in names):
            arrays = [pa.array([None if v is None else bytes(v).decode("latin-1").encode() for v in a.to_pylist()], pa.binary()) if nm == "utf8" else a
                      for nm, a in zip(names, arrays)]
        b = O.batch_from_arrow(pa.RecordBatch.from_arrays(arrays, names=names))
        out.append(S.write_batch(n, b.cols, [True] * len(names) if null_mode == "flag" else None))
    return out


def frame_blocks(raw: bytes, cuts=()) -> bytes:
    """one BlockObject: `raw` cut at the given offsets into `u32 LE length ‖ LZ4 frame` blocks"""
    pts = [0] + list(cuts) + [len(raw)]
    out = b""
    for a, b in zip(pts, pts[1:]):
        fr = pa.Codec("lz4").compress(raw[a:b], asbytes=True)
        out += struct.pack("<I", len(fr)) + fr
    return out


def _canon_oracle(batches, schema):
    cols = []
    for ci, f in enumerate(schema):
        col = []
        for b in batches:
            c = b.cols[ci]
            if f.dtype.id in (T.BINARY,) or f.dtype.id == T.BOOL:
                col += [bytes(v) if f.dtype.id == T.BINARY and ok else (bool(v) if ok else None) for v, ok in zip(c.values, c.valid)]
            else:
                m = S._values_le_bytes(c)
                col += [m[i].tobytes() if ok else None for i, ok in enumerate(c.valid)]
        cols.append(col)
    return cols


def _canon_gpu(batches, schema):
    cols = [[] for _ in schema]
    for rb in batches:
        for ci, f in enumerate(schema):
            a = rb.column(ci)
            if f.dtype.id in (T.BINARY, T.UTF8):
                cols[ci] += [None if v is None else (v.encode() if isinstance(v, str) else v) for v in a.to_pylist()]
            elif f.dtype.id == T.BOOL:
                cols[ci] += a.to_pylist()
            else:
                w = {T.INT8: 1, T.INT16: 2, T.INT32: 4, T.DATE32: 4, T.FLOAT32: 4, T.DECIMAL128: 16}.get(f.dtype.id, 8)
                buf = a.buffers()[1].to_pybytes()[a.offset * w: (a.offset + len(a)) * w]
                valid = a.is_valid().to_pylist()
                cols[ci] += [buf[i * w: (i + 1) * w] if ok else None for i, ok in enumerate(valid)]
    return cols


def _check(read_schema, wire_schema, pushes, conf=None):
    got = PL.collect(PL.IpcReaderExec(read_schema, pushes), conf)
    exp = [b for p in pushes for b in S.read_partition(p, wire_schema)]
    assert _canon_gpu(got, read_schema) == _canon_oracle(exp, wire_schema)
    return got


SIZES = [1] * 33 + [10_000, 3, 10_005, 31, 1, 64, 9_999]               # records start at every bit offset mod 32


@pytest.mark.parametrize("null_mode", ["none", "some", "flag"])
@pytest.mark.parametrize("name", ALL)
def test_round_trip_every_type(name, null_mode):
    rng = np.random.default_rng(ALL.index(name) * 3 + ["none", "some", "flag"].index(null_mode))
    wire, read = _wire_schema(["i64", name] if name != "i64" else [name])
    recs = _records(rng, [f.name for f in wire], SIZES, null_mode)
    pushes = [frame_blocks(b"".join(recs[:20])), frame_blocks(b"".join(recs[20:36]), cuts=[7]), frame_blocks(b"".join(recs[36:]))]
    got = _check(read, wire, pushes, native.default_conf(staging_rows=4096))     # the 10 000-row records are each above staging_rows
    assert sum(b.num_rows for b in got) == sum(SIZES)


def test_all_types_in_one_schema_one_push_and_non_nullable_fields():
    rng = np.random.default_rng(5)
    wire, read = _wire_schema(ALL)
    recs = _records(rng, ALL, [1, 2, 3, 5000, 29, 1, 70_000], "some")
    _check(read, wire, [frame_blocks(b"".join(recs))])
    wire_nn, read_nn = _wire_schema(ALL, nullable=False)
    recs = _records(rng, ALL, [100, 1, 3000], "none")
    got = _check(read_nn, wire_nn, [frame_blocks(b"".join(recs))])
    assert all(c.null_count == 0 for b in got for c in b.columns)


def test_record_straddling_two_blocks_of_one_push():
    rng = np.random.default_rng(9)
    wire, read = _wire_schema(["i64", "bin", "bool", "dec"])
    recs = _records(rng, ["i64", "bin", "bool", "dec"], [3000, 4000, 1, 2], "some")
    raw = b"".join(recs)
    cuts = [1, len(recs[0]) + 17, len(recs[0]) + len(recs[1]) // 2, len(raw) - 3]
    _check(read, wire, [frame_blocks(raw, cuts)])


def test_empty_pushes_and_zero_row_records():
    wire, read = _wire_schema(["i32", "bin"])
    rng = np.random.default_rng(2)
    recs = _records(rng, ["i32", "bin"], [0, 5, 0], "some")
    pushes = [b"", frame_blocks(recs[0]), frame_blocks(b"".join(recs[1:]))]
    got = PL.collect(PL.IpcReaderExec(read, pushes))
    assert sum(b.num_rows for b in got) == 5


# ---- files written by the GPU ShuffleWriterExec and by the oracle ------------------------------------------------------------------
def _partitions(data: bytes, index: bytes):
    offs = struct.unpack("<%dq" % (len(index) // 8), index)
    return [data[offs[i]: offs[i + 1]] for i in range(len(offs) - 1)]


SPECS = [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, "v", T.int64), ("a", E.AGG_AVG, "x", T.float64), ("mx", E.AGG_MAX, "x", T.float64),
         ("sd", E.AGG_SUM, "d", T.decimal128(27, 2))]


def _input(n, seed):
    rng = np.random.default_rng(seed)
    raw = rng.integers(-10**12, 10**12, n)
    return pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 400, n, dtype=np.int64)), pa.array(rng.integers(-3, 4, n).astype(np.int32)),
                                       with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.1), with_nulls(rng, rng.normal(0, 1e6, n), 0.1),
                                       pa.array([decimal.Decimal(int(r)).scaleb(-2) for r in raw], pa.decimal128(17, 2)),
                                       pa.array(rng.integers(0, 100, n, dtype=np.int64))], names=["k1", "k2", "v", "x", "d", "f"])


def _map_side(tmp_path, rb, keys, P, nmaps=3):
    ins = T.from_arrow_schema(rb.schema)
    g = [E.GroupingExpr(k, E.Column(k)) for k in keys]
    preds = [E.BinaryExpr(E.Column("f"), "Lt", E.Literal(70, T.int64))]
    files, n = [], rb.num_rows
    bounds = np.linspace(0, n, nmaps + 1).astype(int)
    for m in range(nmaps):
        leaf = PL.MemoryExec.from_arrow(split_batches(rb.slice(bounds[m], bounds[m + 1] - bounds[m]), 5_000), rb.schema)
        partial = PL.AggExec(PL.HashAgg, g, [E.AggExpr(nm, E.PARTIAL, PL.create_agg(fn, [E.Column(c)], ins, rt)) for nm, fn, c, rt in SPECS], False,
                             PL.FilterExec(preds, leaf))
        w = PL.ShuffleWriterExec(partial, ("hash", [E.Column(k) for k in keys], P), str(tmp_path / f"m{m}.data"), str(tmp_path / f"m{m}.index"))
        PL.collect(w, native.default_conf())
        files.append(_partitions(open(w.output_data_file, "rb").read(), open(w.output_index_file, "rb").read()))
    return ins, g, preds, partial.schema(), files


def _final(ins, pschema):
    by_name = {f.name: f.dtype for f in ins}
    return [E.AggExpr(nm, E.FINAL, PL.create_agg(fn, [E.placeholder(by_name[c])], pschema, rt)) for nm, fn, c, rt in SPECS]


def test_gpu_shuffle_writer_files_partition_by_partition(tmp_path):
    """Binary agg-state columns as the GPU map side writes them, read back through .index"""
    _, _, _, pschema, files = _map_side(tmp_path, _input(30_000, 3), ["k1", "k2"], 13)
    for q in range(13):
        pushes = [f[q] for f in files if f[q]]
        if pushes:
            _check(pschema, pschema, pushes)


def test_oracle_writer_files(tmp_path):
    rng = np.random.default_rng(4)
    wire, read = _wire_schema(["i64", "bin", "f64", "bool", "dec"])
    rb = pa.RecordBatch.from_arrays([_array(rng, nm, 20_000, "some") for nm in ["i64", "bin", "f64", "bool", "dec"]], names=["i64", "bin", "f64", "bool", "dec"])
    batches = [O.batch_from_arrow(b) for b in split_batches(rb, 3000)]
    data, index = S.shuffle_write(batches, S.Partitioning("hash", 5, hash_cols=[0]))
    for part in _partitions(data, index):
        if part:
            _check(read, wire, [part])


# ---- the reduce side end to end --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keys", [["k1"], ["k1", "k2"]])
def test_map_side_then_final_reduce_on_the_gpu(tmp_path, keys):
    """test_map_side_then_final_reduce's plan with the reduce side as IpcReader -> AggExec(Final) over each partition's byte ranges"""
    rb = _input(30_000, 17 + len(keys))
    P = 11
    ins, g, preds, pschema, files = _map_side(tmp_path, rb, keys, P)
    got = []
    for q in range(P):
        pushes = [f[q] for f in files if f[q]]
        if pushes:
            got += PL.collect(PL.AggExec(PL.HashAgg, g, _final(ins, pschema), False, PL.IpcReaderExec(pschema, pushes)))
    op = O.AggExec(E.HASH_AGG, g, [E.AggExpr(nm, E.PARTIAL, PL.create_agg(fn, [E.Column(c)], ins, rt)) for nm, fn, c, rt in SPECS], False, ins)
    of = O.AggExec(E.HASH_AGG, g, _final(ins, op.schema), False, op.schema)
    exp = of.execute(op.execute(O.FilterExec(preds, ins).execute(oracle_batches([rb]))))
    nk = len(keys)
    assert_multiset_equal(got, exp, float_cols=(nk + 2, nk + 3))


def test_final_reduce_then_sort_fetch(tmp_path):
    rb = _input(20_000, 8)
    ins, g, preds, pschema, files = _map_side(tmp_path, rb, ["k1"], 1)
    fin = PL.AggExec(PL.HashAgg, g, _final(ins, pschema), False, PL.IpcReaderExec(pschema, [f[0] for f in files]))
    got = pa.Table.from_batches(PL.collect(PL.SortExec(fin, [(E.Column("s"), True, False), (E.Column("k1"), False, False)], fetch=25)))
    full = pa.Table.from_batches(PL.collect(PL.AggExec(PL.HashAgg, g, _final(ins, pschema), False, PL.IpcReaderExec(pschema, [f[0] for f in files]))))
    rows = sorted(zip(full.column("s").to_pylist(), full.column("k1").to_pylist()), key=lambda t: (-(t[0] if t[0] is not None else -2**70), t[1]))
    assert list(zip(got.column("s").to_pylist(), got.column("k1").to_pylist())) == rows[:25]


def test_hash_join_probe_over_the_reader():
    rng = np.random.default_rng(12)
    wire, read = _wire_schema(["i64", "f64"], nullable=False)
    keys = rng.integers(0, 500, 6000, dtype=np.int64)
    vals = rng.normal(0, 1, 6000)
    rb = pa.RecordBatch.from_arrays([pa.array(keys), pa.array(vals)], names=["i64", "f64"])
    raw = b"".join(S.write_batch(b.num_rows, O.batch_from_arrow(b).cols) for b in split_batches(rb, 1000))
    build_rb = pa.RecordBatch.from_arrays([pa.array(np.arange(0, 500, 2, dtype=np.int64)), pa.array(np.arange(250, dtype=np.int32))], names=["bk", "bv"])
    bs = T.from_arrow_schema(build_rb.schema)
    build = PL.MemoryExec.from_arrow([build_rb])
    probe = PL.IpcReaderExec(read, [frame_blocks(raw, cuts=[len(raw) // 3])])
    schema = PL.build_join_schema(read, bs, PL.JOIN_INNER)
    j = PL.BroadcastJoinExec(schema, probe, build, [(E.Column("i64"), E.Column("bk"))], PL.JOIN_INNER, PL.RIGHT_SIDE)
    got = pa.Table.from_batches(PL.collect(j))
    exp = sorted((int(k), float(v), int(k), int(k) // 2) for k, v in zip(keys, vals) if k % 2 == 0)
    assert sorted(zip(*[got.column(i).to_pylist() for i in range(4)])) == exp


def _device_bytes(ptr, nbytes):
    """bytes [ptr, ptr + nbytes) of device memory, through the CUDA runtime torch has loaded"""
    import ctypes
    cudart = ctypes.CDLL("libcudart.so.12")
    out = ctypes.create_string_buffer(nbytes)
    assert cudart.cudaMemcpy(out, ctypes.c_void_p(ptr), ctypes.c_size_t(nbytes), 2) == 0          # cudaMemcpyDeviceToHost
    return out.raw


def test_device_output_through_pull_device():
    import torch  # noqa: F401  (loads the CUDA runtime)
    rng = np.random.default_rng(3)
    wire, read = _wire_schema(["i64", "bin"])
    recs = _records(rng, ["i64", "bin"], [1000, 1, 2345], "some")
    plan = PL.IpcReaderExec(read, [frame_blocks(b"".join(recs))])
    exp = S.read_partition(plan.batches[0], wire)
    ev = np.concatenate([b.cols[0].values for b in exp]).astype(np.int64)
    valid = np.concatenate([b.cols[0].valid for b in exp])
    with native.NativeOp(plan.plan_bytes()) as op:
        op.push_ipc(plan.batches[0])
        op.finish()
        d = op.pull_device()
        assert d is not None and d.array.length == 3346 and d.device_type == native.ARROW_DEVICE_CUDA
        c0 = d.array.children[0].contents
        off, n = c0.offset, c0.length
        got = np.frombuffer(_device_bytes(c0.buffers[1] + off * 8, n * 8), np.int64)
        bits = np.unpackbits(np.frombuffer(_device_bytes(c0.buffers[0], (off + n + 7) // 8), np.uint8), bitorder="little")[off: off + n].astype(bool)
        assert (bits == valid).all() and (got[valid] == ev[valid]).all()
        native.release_device_array(d)
        assert op.pull_device() is None


# ---- state and validation rules --------------------------------------------------------------------------------------------------
def _status(fn):
    with pytest.raises(native.NativeError) as ei:
        fn()
    return ei.value


def test_push_rules():
    s = Schema([Field("k", T.int64, False)])
    rb = pa.RecordBatch.from_arrays([pa.array([1, 2, 3], pa.int64())], names=["k"])
    with native.NativeOp(PL.IpcReaderExec(s).plan_bytes()) as op:
        assert _status(lambda: op.push(rb)).code == native.ERR_STATE
        op.push_ipc(frame_blocks(S.write_batch(3, O.batch_from_arrow(rb).cols)))
        op.finish()
        assert sum(b.num_rows for b in op.pull_all()) == 3
    with native.NativeOp(PL.MemoryExec(s).plan_bytes()) as op:
        assert _status(lambda: op.push_ipc(b"")).code == native.ERR_STATE


def _bad_pushes():
    good = b"".join(_records(np.random.default_rng(6), ["i32", "bin"], [50, 7], "some"))
    # one record of 50 rows, no NULLs, 1-byte Binary values: n | i32 (flag, 4 x 50 planes) | bin (flag, 4 x 50 length planes, 50 bytes)
    rb = pa.RecordBatch.from_arrays([pa.array(np.arange(50, dtype=np.int32)), pa.array([b"x"] * 50, pa.binary())], names=["i32", "bin"])
    rec = bytearray(S.write_batch(50, O.batch_from_arrow(rb).cols))
    planes = 1 + 1 + 200 + 1
    assert len(rec) == planes + 200 + 50
    past = bytearray(rec); past[planes + 100: planes + 150] = bytes([0x7F] * 50)       # third plane: lengths far past the payload
    neg = bytearray(rec); neg[planes + 150] = 0x80                                     # high plane of row 0: a negative length
    zstd = bytes([0x28, 0xB5, 0x2F, 0xFD]) + bytes(12)
    one_i64 = S.write_batch(4, O.batch_from_arrow(pa.RecordBatch.from_arrays([pa.array([1, 2, 3, 4], pa.int64())], names=["x"])).cols)
    return {
        "truncated record": (frame_blocks(good[:-5]), native.ERR_INVALID_ARG),
        "garbage frame": (struct.pack("<I", 16) + bytes(range(16)), native.ERR_INVALID_ARG),
        "block length past the push": (struct.pack("<I", 1000) + bytes(10), native.ERR_INVALID_ARG),
        "length planes past the payload": (frame_blocks(bytes(past)), native.ERR_INVALID_ARG),
        "negative length": (frame_blocks(bytes(neg)), native.ERR_INVALID_ARG),
        "wrong column layout": (frame_blocks(one_i64), native.ERR_INVALID_ARG),
        "bad null flag": (frame_blocks(S.write_len(3) + b"\x02"), native.ERR_INVALID_ARG),
        "zstd": (struct.pack("<I", len(zstd)) + zstd, native.ERR_UNSUPPORTED),
    }


@pytest.mark.parametrize("name", list(_bad_pushes()))
def test_malformed_pushes_are_refused_and_the_op_stays_usable(name):
    bad, code = _bad_pushes()[name]
    rng = np.random.default_rng(1)
    wire, read = _wire_schema(["i32", "bin"])
    good = _records(rng, ["i32", "bin"], [10, 20], "some")
    with native.NativeOp(PL.IpcReaderExec(read).plan_bytes()) as op:
        op.push_ipc(frame_blocks(good[0]))
        e = _status(lambda: op.push_ipc(bad))
        assert e.code == code and "push_ipc" in e.msg, e.msg
        op.push_ipc(frame_blocks(good[1]))                                 # nothing of the refused push was kept
        op.finish()
        got = op.pull_all()
    exp = [b for p in good for b in S.read_partition(frame_blocks(p), wire)]
    assert _canon_gpu(got, read) == _canon_oracle(exp, wire)
