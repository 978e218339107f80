"""ShuffleWriterExec over batches with Binary columns (the reference-format AggExec(Partial) output: grouping columns plus one
Binary column of frozen accumulator rows) through the C ABI vs the oracle (oracle/shuffle_oracle.py).  The files are read back
the way the reduce side does; every partition must hold exactly the rows pmod(murmur3(keys, 42), P) sends there (as a multiset),
every record must re-encode to the same bytes with the oracle's write_batch, and the chunks must be what the files frame."""
import decimal
import os
import struct

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from oracle import blaze_oracle as O
from oracle import shuffle_oracle as S
from helpers import *

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _zeroed(rng, values, null_frac, pa_type=None):
    """NULL slots hold 0, as the oracle's writer stores them, so records re-encode byte for byte"""
    if null_frac <= 0:
        return pa.array(values, type=pa_type)
    mask = rng.random(len(values)) < null_frac
    return pa.array(np.where(mask, 0, values).astype(values.dtype), mask=mask, type=pa_type)


def _binary(rng, n, null_frac, huge=False):
    """0-byte values, 1-32 bytes, 64-300 bytes (every alignment of source and destination), optionally one of 1 MiB + 3"""
    kind = rng.random(n)
    lens = np.where(kind < 0.1, 0, np.where(kind < 0.9, rng.integers(1, 33, n), rng.integers(64, 301, n)))
    pool = rng.integers(0, 256, int(lens.sum()) + 1, dtype=np.uint8).tobytes()
    out, pos = [], 0
    for i, ln in enumerate(lens):
        out.append(None if rng.random() < null_frac else pool[pos: pos + int(ln)])
        pos += int(ln)
    if huge and n:
        out[n // 2] = bytes(rng.integers(0, 256, (1 << 20) + 3, dtype=np.uint8))
    return pa.array(out, pa.binary())


def _table(n, seed, nbin, null_frac, huge=False):
    rng = np.random.default_rng(seed)
    cols = {"k": _zeroed(rng, rng.integers(-50, 5000, n, dtype=np.int64), null_frac / 4),
            "b0": _binary(rng, n, null_frac, huge),
            "i": _zeroed(rng, rng.integers(-2**31, 2**31, n).astype(np.int32), null_frac, pa.int32()),
            "dec": pa.array([decimal.Decimal(int(x)).scaleb(-2) for x in rng.integers(-10**15, 10**15, n)], pa.decimal128(20, 2),
                            mask=(rng.random(n) < null_frac) if null_frac else None),
            "flag": pa.array(rng.random(n) < 0.3, pa.bool_())}
    for j in range(1, nbin):
        cols[f"b{j}"] = _binary(rng, n, null_frac)
    names = list(cols)
    fields = [pa.field(c, cols[c].type, c != "flag") for c in names]
    return pa.RecordBatch.from_arrays([cols[c] for c in names], schema=pa.schema(fields))


def _records(raw, schema):
    """(decoded batch, its bytes) of every record in `raw`"""
    out, pos = [], 0
    while pos < len(raw):
        b, end = S.read_batch(raw, pos, schema)
        out.append((b, raw[pos:end]))
        pos = end
    return out


def _check_files(plan, batches, keys, P, max_rows=None):
    data = open(plan.output_data_file, "rb").read()
    index = open(plan.output_index_file, "rb").read()
    assert len(index) == 8 * (P + 1)
    offs = struct.unpack("<%dq" % (P + 1), index)
    assert offs[0] == 0 and offs[-1] == len(data) and all(a <= b for a, b in zip(offs, offs[1:]))
    schema = T.from_arrow_schema(batches[0].schema)
    whole = O.concat_batches(schema, oracle_batches(batches))
    hash_cols = [batches[0].schema.names.index(k) for k in keys]
    pid = S.evaluate_partition_ids(S.Partitioning("hash", P, hash_cols=hash_cols), whole) if P > 1 else np.zeros(whole.num_rows, np.uint32)
    nullable = [f.nullable for f in schema]
    total = 0
    for q in range(P):
        raw = S.read_ipc_blocks(data[offs[q]: offs[q + 1]])
        assert raw == b"".join(ch["data"][ch["part_off"][q]: ch["part_off"][q + 1]] for ch in plan.last_chunks)
        recs = _records(raw, schema)
        for b, rec in recs:                                   # length planes, data order and flags pin the bytes
            assert 0 < b.num_rows and (max_rows is None or b.num_rows <= max_rows)
            assert S.write_batch(b.num_rows, b.cols, has_nulls=nullable) == rec
        exp = whole.take(np.nonzero(pid == q)[0])
        assert O.rows_multiset([b for b, _ in recs]) == O.rows_multiset([exp]), f"partition {q}"
        if exp.num_rows == 0:
            assert offs[q] == offs[q + 1]
        total += sum(b.num_rows for b, _ in recs)
    assert total == whole.num_rows
    assert sum(ch["rows"] for ch in plan.last_chunks) == whole.num_rows


def _shuffle(tmp_path, batches, keys, P, conf):
    leaf = PL.MemoryExec.from_arrow(batches, batches[0].schema)
    part = ("hash", [E.Column(k) for k in keys], P) if P > 1 else ("single",)
    plan = PL.ShuffleWriterExec(leaf, part, str(tmp_path / "s.data"), str(tmp_path / "s.index"))
    assert PL.collect(plan, conf) == []
    return plan


@pytest.mark.parametrize("P,nbin,keys", [(1, 1, []), (7, 2, ["k"]), (200, 3, ["k", "i"]), (4096, 1, ["dec", "flag"])])
@pytest.mark.parametrize("batch_size", [64, 10000])
@pytest.mark.parametrize("null_frac", [0.0, 0.2])
def test_mixed_schemas(tmp_path, P, nbin, keys, batch_size, null_frac):
    rb = _table(6_000, 31 + P + nbin, nbin, null_frac, huge=(P == 7 and batch_size == 64))
    batches = split_batches(rb, 2_500)
    plan = _shuffle(tmp_path, batches, keys, P, native.default_conf(staging_rows=0, batch_size=batch_size))
    assert plan.last_metrics["fast_path_launches"] == len(batches)
    _check_files(plan, batches, keys, P, max_rows=max(20, batch_size))


def test_all_empty_and_all_null_binary(tmp_path):
    n = 3_000
    rng = np.random.default_rng(4)
    rb = pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 100, n, dtype=np.int64)), pa.array([b""] * n, pa.binary()), pa.array([None] * n, pa.binary())],
                                    schema=pa.schema([pa.field("k", pa.int64(), False), pa.field("e", pa.binary(), False), pa.field("z", pa.binary(), True)]))
    plan = _shuffle(tmp_path, [rb], ["k"], 13, native.default_conf(staging_rows=0))
    _check_files(plan, [rb], ["k"], 13)


def test_several_chunks_and_staged_host_batches(tmp_path):
    """a small max_launch_rows cuts every pushed batch into several chunks (each with its own rows per record); 10,000-row host
    batches go through the pinned staging ring"""
    rb = _table(40_000, 7, 2, 0.1)
    batches = split_batches(rb, 10_000)
    plan = _shuffle(tmp_path, batches, ["k"], 50, native.default_conf(staging_rows=1 << 15))
    _check_files(plan, batches, ["k"], 50)
    plan = _shuffle(tmp_path, batches, ["k"], 50, native.default_conf(staging_rows=0, max_launch_rows=3_000))
    assert len(plan.last_chunks) == 4 * 4
    _check_files(plan, batches, ["k"], 50)


def _device_batch(rb, torch, offset=0, length=None, base_shift=0):
    """device copies of rb's buffers; Binary offsets are shifted by base_shift (the data buffer gets that many leading bytes), and the
    children carry the Arrow offset `offset` (length rows from there)"""
    cols, keep = [], []
    for c in rb.columns:
        assert c.offset == 0
        valid = torch.tensor(np.frombuffer(c.buffers()[0], np.uint8).copy(), device="cuda") if c.null_count else None
        if pa.types.is_binary(c.type):
            offs = np.frombuffer(c.buffers()[1], np.int32)[: len(c) + 1].astype(np.int32) + base_shift
            raw = np.frombuffer(c.buffers()[2], np.uint8) if c.buffers()[2] is not None else np.zeros(0, np.uint8)
            data = torch.tensor(np.concatenate([np.full(base_shift, 0xEE, np.uint8), raw, np.zeros(16, np.uint8)]), device="cuda")
            to = torch.tensor(offs, device="cuda")
            cols.append((data.data_ptr(), valid.data_ptr() if valid is not None else 0, len(c), to.data_ptr()))
            keep += [to, data]
        elif pa.types.is_boolean(c.type):
            v = torch.tensor(np.frombuffer(c.buffers()[1], np.uint8).copy(), device="cuda")
            cols.append((v.data_ptr(), valid.data_ptr() if valid is not None else 0, len(c))); keep.append(v)
        else:
            v = torch.tensor(c.fill_null(0).to_numpy(zero_copy_only=False), device="cuda")
            cols.append((v.data_ptr(), valid.data_ptr() if valid is not None else 0, len(c))); keep.append(v)
        if valid is not None:
            keep.append(valid)
    db = native.DeviceBatch(cols, rb.num_rows, 0, keep)
    if offset or length is not None:
        for i in range(db.n):
            db.children[i].offset = offset
            db.children[i].length = length
        db.dev.array.length = length
    return db


def test_sliced_device_input(tmp_path):
    """push_device with an Arrow offset != 0 and offsets[0] != 0 (borrowed caller memory)"""
    torch = pytest.importorskip("torch")
    rb = pa.RecordBatch.from_arrays([pa.array(np.arange(9_000, dtype=np.int64)), _binary(np.random.default_rng(5), 9_000, 0.15)],
                                    schema=pa.schema([pa.field("k", pa.int64(), False), pa.field("b", pa.binary(), True)]))
    schema = T.from_arrow_schema(rb.schema)
    plan = PL.ShuffleWriterExec(PL.MemoryExec(schema), ("hash", [E.Column("k")], 31), str(tmp_path / "s.data"), str(tmp_path / "s.index"))
    with native.NativeOp(plan.plan_bytes(), native.default_conf(staging_rows=0)) as op:
        op.push_device(_device_batch(rb, torch, offset=1_234, length=6_000, base_shift=37))
        op.finish()
        plan.last_chunks = op.shuffle_chunks()
    _check_files(plan, [rb.slice(1_234, 6_000)], ["k"], 31)


def test_committed_partial_state_fixture(tmp_path):
    """the reference-format AggExec(Partial) output of tests/golden (grouping key + frozen SUM/COUNT rows) shuffled and read back
    unchanged"""
    with pa.ipc.open_file(os.path.join(GOLDEN, "m1_sum_count_partial.out.arrow")) as f:
        tbl = f.read_all()
    batches = tbl.to_batches()
    assert pa.types.is_binary(tbl.schema.field(tbl.num_columns - 1).type)
    for P, keys in ((1, []), (9, [tbl.schema.names[0]])):
        plan = _shuffle(tmp_path, batches, keys, P, native.default_conf(staging_rows=0))
        _check_files(plan, batches, keys, P)


# ---- the map / reduce split of an aggregation query --------------------------------------------------------------------------
SPECS = [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, "v", T.int64), ("a", E.AGG_AVG, "x", T.float64), ("mn", E.AGG_MIN, "v", T.int64),
         ("mx", E.AGG_MAX, "x", T.float64), ("sd", E.AGG_SUM, "d", T.decimal128(27, 2)), ("ad", E.AGG_AVG, "d", T.decimal128(21, 6)),
         ("md", E.AGG_MAX, "d", T.decimal128(17, 2))]


@pytest.mark.parametrize("keys", [["k1"], ["k1", "k2"]])
def test_map_side_then_final_reduce(tmp_path, keys):
    """three map tasks: Filter -> AggExec(Partial, reference format) -> ShuffleWriterExec over their own slices; per reduce partition,
    GPU AggExec(Final) over that partition of every map output; the union equals one group-by over the whole input"""
    rng = np.random.default_rng(17 + len(keys))
    n, P = 30_000, 11
    raw = rng.integers(-10**12, 10**12, n)
    rb = pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 400, n, dtype=np.int64)), pa.array(rng.integers(-3, 4, n).astype(np.int32)),
                                     with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.1), with_nulls(rng, rng.normal(0, 1e6, n), 0.1),
                                     pa.array([decimal.Decimal(int(r)).scaleb(-2) for r in raw], pa.decimal128(17, 2)),
                                     pa.array(rng.integers(0, 100, n, dtype=np.int64))], names=["k1", "k2", "v", "x", "d", "f"])
    ins = T.from_arrow_schema(rb.schema)
    g = [E.GroupingExpr(k, E.Column(k)) for k in keys]
    preds = [E.BinaryExpr(E.Column("f"), "Lt", E.Literal(70, T.int64))]

    def partial_of(leaf):
        return PL.AggExec(PL.HashAgg, g, [E.AggExpr(nm, E.PARTIAL, PL.create_agg(fn, [E.Column(c)], ins, rt)) for nm, fn, c, rt in SPECS], False,
                          PL.FilterExec(preds, leaf))

    maps = []
    for m, (lo, hi) in enumerate(((0, 9_000), (9_000, 21_000), (21_000, n))):
        leaf = PL.MemoryExec.from_arrow(split_batches(rb.slice(lo, hi - lo), 5_000), rb.schema)
        partial = partial_of(leaf)
        w = PL.ShuffleWriterExec(partial, ("hash", [E.Column(k) for k in keys], P), str(tmp_path / f"m{m}.data"), str(tmp_path / f"m{m}.index"))
        PL.collect(w, native.default_conf())                                   # default conf: partial state in the reference format
        maps.append(S.read_shuffle_file(open(w.output_data_file, "rb").read(), open(w.output_index_file, "rb").read(), partial.schema()))
    pschema = partial.schema()
    got = []
    for q in range(P):
        parts = [O.batch_to_arrow(b) for mp in maps for b in mp[q]]
        if not parts:
            continue
        fin = PL.AggExec(PL.HashAgg, g, _final(SPECS, ins, pschema), False, PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(pschema)))
        got += PL.collect(fin)
    whole = oracle_batches([rb])
    op = O.AggExec(E.HASH_AGG, g, [E.AggExpr(nm, E.PARTIAL, PL.create_agg(fn, [E.Column(c)], ins, rt)) for nm, fn, c, rt in SPECS], False, ins)
    of = O.AggExec(E.HASH_AGG, g, _final(SPECS, ins, op.schema), False, op.schema)
    exp = of.execute(op.execute(O.FilterExec(preds, ins).execute(whole)))
    nk = len(keys)
    assert_multiset_equal(got, exp, float_cols=(nk + 2, nk + 4))


def _final(specs, ins, pschema):
    by_name = {f.name: f.dtype for f in ins}
    return [E.AggExpr(nm, E.FINAL, PL.create_agg(fn, [E.placeholder(by_name[c])], pschema, rt)) for nm, fn, c, rt in specs]


# ---- limits and refusals ------------------------------------------------------------------------------------------------------
def test_binary_hash_keys_and_utf8_columns_are_refused(tmp_path):
    rb = pa.RecordBatch.from_arrays([pa.array(np.arange(10, dtype=np.int64)), pa.array([b"x"] * 10, pa.binary()), pa.array(["s"] * 10, pa.string())],
                                    names=["k", "b", "s"])
    def refused(batch, keys):
        plan = PL.ShuffleWriterExec(PL.MemoryExec.from_arrow([batch]), ("hash", [E.Column(k) for k in keys], 4), str(tmp_path / "d"), str(tmp_path / "i"))
        with pytest.raises(native.NativeError) as ei:
            PL.collect(plan)
        assert ei.value.code == native.ERR_UNSUPPORTED
        return ei.value.msg
    assert "binary" in refused(rb.select([0, 1]), ["b"]).lower()
    assert "shuffle" in refused(rb, ["k"])


def test_large_batch_record_over_int32_is_refused(tmp_path):
    """two Binary columns of six 200 MiB values each, P = 1: one record would carry 2.5 GB of Binary data, more than 2^31 - 1 bytes
    -> UNSUPPORTED, nothing truncated"""
    torch = pytest.importorskip("torch")
    n, each = 6, 200 << 20
    k = torch.arange(n, dtype=torch.int64, device="cuda")
    cols, keep = [(k.data_ptr(), 0, n)], [k]
    for _ in range(2):
        data = torch.zeros(n * each + 16, dtype=torch.uint8, device="cuda")
        offs = torch.arange(0, n + 1, dtype=torch.int64, device="cuda").mul(each).to(torch.int32)
        cols.append((data.data_ptr(), 0, n, offs.data_ptr())); keep += [data, offs]
    schema = T.Schema([T.Field("k", T.int64, False), T.Field("b0", T.binary, False), T.Field("b1", T.binary, False)])
    plan = PL.ShuffleWriterExec(PL.MemoryExec(schema), ("single",), str(tmp_path / "s.data"), str(tmp_path / "s.index"))
    torch.cuda.synchronize()                                   # the buffers are written on torch's stream; the op reads them on its own
    with native.NativeOp(plan.plan_bytes(), native.default_conf(staging_rows=0)) as op:
        with pytest.raises(native.NativeError) as ei:
            op.push_device(native.DeviceBatch(cols, n, 0, keep))
            op.finish()
    assert ei.value.code == native.ERR_UNSUPPORTED and "INT32_MAX" in ei.value.msg


def _copy_device_range(ptr, nbytes):
    """bytes [ptr, ptr + nbytes) of device memory, through the CUDA runtime torch has loaded"""
    import ctypes
    cudart = ctypes.CDLL("libcudart.so.12")
    out = ctypes.create_string_buffer(nbytes)
    assert cudart.cudaMemcpy(out, ctypes.c_void_p(ptr), ctypes.c_size_t(nbytes), 2) == 0          # cudaMemcpyDeviceToHost
    return out.raw


def test_large_batch_chunk_over_4gib_on_device(tmp_path):
    """three Binary columns of ~1.5 GiB each in one chunk (> 2^32 data bytes), kept on the device: part_off is right and every record
    decodes to its rows"""
    torch = pytest.importorskip("torch")
    n, each, P = 24_000, 65_536 + 7, 3
    k = torch.arange(n, dtype=torch.int64, device="cuda")
    cols, keep = [(k.data_ptr(), 0, n)], [k]
    for j in range(3):
        data = torch.arange(n * each + 16, dtype=torch.int32, device="cuda").add_(j * 7919).remainder_(251).to(torch.uint8)
        offs = torch.arange(0, n + 1, dtype=torch.int64, device="cuda").mul(each).to(torch.int32)
        cols.append((data.data_ptr(), 0, n, offs.data_ptr())); keep += [data, offs]
    schema = T.Schema([T.Field("k", T.int64, False)] + [T.Field(f"b{j}", T.binary, False) for j in range(3)])
    plan = PL.ShuffleWriterExec(PL.MemoryExec(schema), ("hash", [E.Column("k")], P), str(tmp_path / "s.data"), str(tmp_path / "s.index"))
    torch.cuda.synchronize()                                   # the buffers are written on torch's stream; the op reads them on its own
    with native.NativeOp(plan.plan_bytes(), native.default_conf(staging_rows=0, shuffle_output_on_device=1)) as op:
        op.push_device(native.DeviceBatch(cols, n, 0, keep))
        op.finish()
        (ch,) = op.shuffle_chunks()
        assert ch["on_device"] and ch["rows"] == n and sum(ch["part_rows"]) == n
        off = ch["part_off"]
        assert off[-1] > 1 << 32 and all(a <= b for a, b in zip(off, off[1:]))
        whole = O.Batch(T.Schema([T.Field("k", T.int64, False)]), [O.Col(T.int64, np.arange(n, dtype=np.int64), np.ones(n, bool))], n)
        pid = S.evaluate_partition_ids(S.Partitioning("hash", P, hash_cols=[0]), whole)
        data_bytes = 0
        for q in range(P):
            assert ch["part_rows"][q] == int((pid == q).sum())
            host = _copy_device_range(ch["data_ptr"] + off[q], off[q + 1] - off[q])
            pos, rows = 0, 0
            while pos < len(host):
                b, pos = S.read_batch(host, pos, schema)
                ks = b.cols[0].values
                assert (pid[ks] == q).all()
                for j in range(3):
                    vals = b.cols[j + 1].values
                    assert all(len(v) == each for v in vals)
                    for r in (0, len(vals) - 1):
                        start = int(ks[r]) * each + j * 7919
                        assert vals[r] == (np.arange(start, start + each, dtype=np.int64) % 251).astype(np.uint8).tobytes()
                    data_bytes += each * len(vals)
                rows += b.num_rows
            assert rows == ch["part_rows"][q]
        assert data_bytes == 3 * n * each
