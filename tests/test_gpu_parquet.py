"""ParquetScanExec on the GPU (SURVEY.md §8(f) rank 3) through the C ABI.  The decode arithmetic of the reference lives in the
un-vendored `parquet` 55.2 crate and no native test of the reference pins it (SURVEY §8f-3: "parity unpinned"), so the oracle is
a second engine: pyarrow's libparquet reads the same files — values, NULLs and row order must match exactly.  Files are written
here with every page shape the GPU path decodes: PLAIN / RLE_DICTIONARY (incl. dictionary fallback), data page v1 / v2,
UNCOMPRESSED / SNAPPY, required / optional columns, several row groups."""
import ctypes as C
import decimal
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from helpers import *

pytestmark = pytest.mark.gpu


def _table(n, seed, null_frac):
    rng = np.random.default_rng(seed)
    m = lambda: (rng.random(n) < null_frac) if null_frac else None
    cols = {
        "k": pa.array(np.sort(rng.integers(0, 10_000, n, dtype=np.int64))),                      # sorted: row-group statistics can prune
        "i64": pa.array(rng.integers(-2**62, 2**62, n, dtype=np.int64), mask=m()),
        "i32": pa.array(rng.integers(-50, 50, n).astype(np.int32), pa.int32(), mask=m()),          # few distinct values: dictionary pages
        "i16": pa.array(rng.integers(-2**15, 2**15, n).astype(np.int16), pa.int16(), mask=m()),
        "i8": pa.array(rng.integers(-128, 128, n).astype(np.int8), pa.int8(), mask=m()),
        "f32": pa.array(rng.normal(size=n).astype(np.float32), pa.float32(), mask=m()),
        "f64": pa.array(rng.normal(0, 1e9, n), mask=m()),
        "d": pa.array(rng.integers(0, 20000, n).astype(np.int32), pa.int32(), mask=m()).cast(pa.date32()),
        "ts": pa.array(rng.integers(0, 2**50, n, dtype=np.int64), mask=m()).cast(pa.timestamp("us")),
        "dec9": pa.array([decimal.Decimal(int(x)).scaleb(-2) for x in rng.integers(-10**8, 10**8, n)], pa.decimal128(9, 2), mask=m()),
        "dec18": pa.array([decimal.Decimal(int(x)).scaleb(-4) for x in rng.integers(-10**17, 10**17, n)], pa.decimal128(18, 4), mask=m()),
        "dec30": pa.array([decimal.Decimal(int(x) * 10**9 + 7).scaleb(-5) for x in rng.integers(-10**17, 10**17, n)], pa.decimal128(30, 5), mask=m()),
        "b": pa.array(rng.random(n) < 0.3, pa.bool_(), mask=m()),
    }
    fields = [pa.field(c, cols[c].type, c != "k") for c in cols]
    return pa.Table.from_arrays(list(cols.values()), schema=pa.schema(fields))


@pytest.mark.parametrize("compression", ["none", "snappy"])
@pytest.mark.parametrize("dictionary", [True, False])
@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
def test_scan_matches_libparquet(tmp_path, compression, dictionary, page_version):
    t = _table(25_000, 3, 0.12)
    path = str(tmp_path / "t.parquet")
    pq.write_table(t, path, compression=compression, use_dictionary=dictionary, data_page_version=page_version, row_group_size=9_000, data_page_size=16 * 1024,
                   store_decimal_as_integer=True)
    plan = parquet_scan(path, t.schema)
    out = PL.collect(plan)
    assert_same_table(out, pq.read_table(path))
    assert plan.last_metrics["gpu_kernel_launches"] > 0 and plan.last_metrics["input_batches"] == 3          # one device batch per row group


def test_required_columns_dictionary_fallback_and_flba_decimals(tmp_path):
    """no NULLs anywhere (no definition levels), a dictionary that overflows into PLAIN pages mid-chunk, decimals stored as FIXED_LEN_BYTE_ARRAY"""
    rng = np.random.default_rng(5)
    n = 120_000
    t = pa.table({"a": pa.array(rng.integers(0, 2**40, n, dtype=np.int64)),                        # ~unique: the dictionary page limit is hit -> PLAIN fallback
                  "d": pa.array([decimal.Decimal(int(x)).scaleb(-3) for x in rng.integers(-10**11, 10**11, n)], pa.decimal128(12, 3)),
                  "c": pa.array((np.arange(n) % 7).astype(np.int32), pa.int32())})
    t = t.cast(pa.schema([pa.field(f.name, f.type, False) for f in t.schema]))
    path = str(tmp_path / "t.parquet")
    pq.write_table(t, path, compression="snappy", use_dictionary=True, dictionary_pagesize_limit=64 * 1024, row_group_size=50_000)
    assert_same_table(PL.collect(parquet_scan(path, t.schema)), pq.read_table(path))


def test_projection_pruning_limit_and_filter_above(tmp_path):
    t = _table(40_000, 8, 0.1)
    path = str(tmp_path / "t.parquet")
    pq.write_table(t, path, compression="snappy", row_group_size=5_000, store_decimal_as_integer=True)
    names = t.schema.names
    proj = [names.index("f64"), names.index("k"), names.index("i32")]
    # projection (subset + reorder)
    assert_same_table(PL.collect(parquet_scan(path, t.schema, projection=proj)), pq.read_table(path, columns=["f64", "k", "i32"]))
    # row-group pruning: k is sorted, 8 row groups; `k >= v` must skip the row groups below v, the FilterExec above removes the rest
    v = int(t.column("k")[22_000].as_py())
    pred = E.BinaryExpr(E.Column("k"), "GtEq", E.Literal(v, T.int64))
    scan = parquet_scan(path, t.schema, projection=proj, pruning_predicates=[pred])
    plan = PL.FilterExec([pred], scan)
    out = PL.collect(plan)
    exp = pq.read_table(path, columns=["f64", "k", "i32"]).filter(pc.field("k") >= v)
    assert_same_table(out, exp)
    m = plan.last_metrics
    assert m["input_batches"] < 8 and m["fast_path_launches"] >= 3, m                                   # pruned row groups never reach the device
    # ScanLimit
    lim = PL.collect(parquet_scan(path, t.schema, projection=proj, limit=7_500))
    assert_same_table(lim, pq.read_table(path, columns=["f64", "k", "i32"]).slice(0, 7_500))
    # an aggregate straight over the scan: the q1 leaf
    ins = scan.schema()
    g = [E.GroupingExpr("i32", E.Column("i32"))]
    mk = lambda mode, ch: [E.AggExpr("c", mode, PL.create_agg(E.AGG_COUNT, ch, ins, T.int64))]
    partial = PL.AggExec(PL.HashAgg, g, mk(E.PARTIAL, [E.Column("k")]), False, parquet_scan(path, t.schema, projection=proj))
    final = PL.AggExec(PL.HashAgg, g, mk(E.FINAL, [E.placeholder(T.int64)]), False, partial)
    got = {(r["i32"], r["c"]) for b in PL.collect(final) for r in b.to_pylist()}
    exp = pq.read_table(path, columns=["i32", "k"]).group_by("i32").aggregate([("k", "count")]).to_pylist()
    assert got == {(r["i32"], r["k_count"]) for r in exp}


def test_splits_cover_every_row_group_once_and_missing_columns_are_null(tmp_path):
    t = _table(30_000, 9, 0.05)
    path = str(tmp_path / "t.parquet")
    pq.write_table(t, path, compression="none", row_group_size=4_000, store_decimal_as_integer=True)
    size = os.path.getsize(path)
    parts = []
    for lo, hi in ((0, size // 3), (size // 3, 2 * size // 3), (2 * size // 3, size)):
        parts += PL.collect(parquet_scan(path, t.schema, range=(lo, hi)))
    assert_same_table(parts, pq.read_table(path))
    wider = pa.schema(list(t.schema) + [pa.field("new_col", pa.int64(), True)])                      # schema evolution: the file predates the column
    out = PL.collect(parquet_scan(path, wider, projection=[0, len(t.schema)]))
    got = pa.Table.from_batches(out)
    assert got.column("new_col").null_count == 30_000 and got.column("k").equals(pq.read_table(path).column("k"))


def test_reader_callback_and_unsupported_shapes(tmp_path):
    t = _table(5_000, 2, 0.1)
    path = str(tmp_path / "t.parquet")
    pq.write_table(t, path, compression="snappy", store_decimal_as_integer=True)
    data = open(path, "rb").read()
    calls = []
    @C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.POINTER(C.c_uint8))
    def reader(ctx, p, off, length, dst):
        calls.append((p.decode(), off, length))
        C.memmove(dst, data[off: off + length], length)
        return 0
    native.check(native.lib.b200q_set_file_reader(C.cast(reader, C.c_void_p), None))
    try:
        plan = PL.ParquetScanExec(T.from_arrow_schema(t.schema), [("hdfs://nn/warehouse/t.parquet", len(data), None)])
        assert_same_table(PL.collect(plan), pq.read_table(path))
        assert calls and all(c[0] == "hdfs://nn/warehouse/t.parquet" for c in calls)
    finally:
        native.check(native.lib.b200q_set_file_reader(None, None))
    # zstd pages and string columns are outside the GPU path: UNSUPPORTED, the host keeps its CPU scan
    pq.write_table(t, path, compression="zstd", store_decimal_as_integer=True)
    with pytest.raises(native.NativeError) as ei:
        PL.collect(parquet_scan(path, t.schema))
    assert ei.value.code == native.ERR_UNSUPPORTED
