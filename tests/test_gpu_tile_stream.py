"""The streaming front end of the tile aggregate kernels (kernels_tile.cu): lane l of a warp holds rows l + 32 j of a 128-row
tile, the filter columns are read first and the key / argument columns only for the rows that pass, and the next tile's
filter columns are in flight while a tile is reduced.  Every case takes a tile kernel and is checked against the oracle:
ragged tails, 8-byte (not 16-byte) aligned device columns, several launches per batch, extreme and clustered selectivities,
filter columns shared with a key or an argument, NULLs at non-zero bit offsets, narrow keys, COUNT(col), the wide kernel's
f64 / decimal / MIN / MAX arguments, and keys that leave the dense range until the hashed table grows (deferred rows)."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
from oracle import blaze_oracle as O
from helpers import *

pytestmark = pytest.mark.gpu

D172 = pa.decimal128(17, 2)


def _table(n, seed, runs=False, null_frac=0.0, key_type=pa.int64(), dec=False):
    """f uniform in [0, 1000) (runs: constant over runs of 8 rows), so that `f BETWEEN 200 AND 399` keeps 20 % of the rows"""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 1000, (n + 7) // 8 if runs else n, dtype=np.int64)
    if runs:
        f = np.repeat(f, 8)[:n]
    k1 = rng.integers(0, 50, n).astype(key_type.to_pandas_dtype())
    k2 = rng.integers(0, 7, n, dtype=np.int64)
    v = rng.integers(-10**9, 10**9, n, dtype=np.int64)
    g = rng.integers(0, 10, n, dtype=np.int64)
    cols = {"f": with_nulls(rng, f, null_frac), "k1": with_nulls(rng, k1, null_frac, key_type), "k2": pa.array(k2),
            "v": with_nulls(rng, v, null_frac), "g": pa.array(g), "x": with_nulls(rng, rng.normal(0, 1e6, n), null_frac)}
    if dec:
        raw = rng.integers(-10**15, 10**15, n)
        cols["d"] = pa.array([decimal.Decimal(int(r)).scaleb(-2) for r in raw], type=D172, mask=(rng.random(n) < null_frac) if null_frac else None)
    names = list(cols)
    return pa.RecordBatch.from_arrays([cols[c] for c in names], names=names)


def _between(col, lo, hi):
    return [E.BinaryExpr(E.Column(col), "GtEq", E.Literal(lo, T.int64)), E.BinaryExpr(E.Column(col), "LtEq", E.Literal(hi, T.int64))]


Q1 = _between("f", 200, 399)


def _aggs(specs, mode, src):
    return [E.AggExpr(nm, mode, PL.create_agg(fn, ([E.Column(col)] if col else [E.Literal(1, T.int64)]) if mode == E.PARTIAL else [E.placeholder(rt)], src, rt))
            for nm, fn, col, rt in specs]


SUM_V = [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, None, T.int64)]


def _check(batches, preds, keys, specs, conf=None, float_cols=(), push=None):
    """Partial -> Final through the C ABI vs the oracle; the Partial stage must have taken a tile kernel"""
    schema = batches[0].schema
    leaf = PL.MemoryExec.from_arrow(batches, schema)
    ins = leaf.schema()
    groupings = [E.GroupingExpr(k, E.Column(k)) for k in keys]
    partial = PL.AggExec(PL.HashAgg, groupings, _aggs(specs, E.PARTIAL, ins), False, PL.FilterExec(preds, leaf) if preds else leaf)
    conf = conf or native.default_conf(staging_rows=0)
    if push is None:
        mid = PL.collect(partial, conf)
        launches = partial.last_metrics["fast_path_launches"]
    else:                                                            # device input: push the device batches by hand
        with native.NativeOp(partial.plan_bytes(), conf) as op:
            for db in push:
                op.push_device(db)
            op.finish()
            mid = op.pull_all()
            launches = op.metrics()["fast_path_launches"]
    assert launches > 0, "the plan must take a tile kernel"
    final = PL.AggExec(PL.HashAgg, groupings, _aggs(specs, E.FINAL, partial.schema()), False, PL.MemoryExec(partial.schema(), mid))
    got = PL.collect(final, conf)
    ob = oracle_batches(batches)
    op_ = O.AggExec(E.HASH_AGG, groupings, _aggs(specs, E.PARTIAL, ins), False, ins)
    of = O.AggExec(E.HASH_AGG, groupings, _aggs(specs, E.FINAL, op_.schema), False, op_.schema)
    exp = of.execute(op_.execute(O.FilterExec(preds, ins).execute(ob) if preds else ob))
    assert_multiset_equal(got, exp, tuple(len(keys) + c for c in float_cols))


@pytest.mark.parametrize("tail", [1, 31, 63, 64, 127])
def test_ragged_tails(tail):
    rb = _table(128 * 37 + tail, 1)
    _check([rb, rb.slice(5, 128 + tail)], Q1, ["k1", "k2"], SUM_V)


def test_several_launches_per_batch():
    rb = _table(300_001, 2)
    _check([rb], Q1, ["k1", "k2"], SUM_V, conf=native.default_conf(staging_rows=0, max_launch_rows=(1 << 16) + 37))


@pytest.mark.parametrize("sel", ["none", "one row", "all", "runs of 8", "0.01", "0.5"])
def test_selectivity(sel):
    if sel == "none":
        rb, preds = _table(20_000, 3), _between("f", 5000, 6000)
    elif sel == "one row":
        rb = _table(20_000, 3)
        f = np.full(20_000, 0, dtype=np.int64); f[12_345] = 300
        rb = rb.set_column(0, "f", pa.array(f))
        preds = Q1
    elif sel == "all":
        rb, preds = _table(20_000, 3), _between("f", 0, 999)
    elif sel == "runs of 8":
        rb, preds = _table(20_000, 3, runs=True), Q1
    else:
        rb, preds = _table(20_000, 3), _between("f", 200, 200 + int(1000 * float(sel)) - 1)
    _check(split_batches(rb, 7_000), preds, ["k1", "k2"], SUM_V)


@pytest.mark.parametrize("shape", ["two filter columns", "filter on the key", "filter on the argument", "filter on both keys"])
def test_shared_and_two_filter_columns(shape):
    rb = _table(30_000, 4)
    preds = {"two filter columns": Q1 + _between("g", 2, 8),
             "filter on the key": Q1 + _between("k1", 3, 40),
             "filter on the argument": _between("v", -10**8, 5 * 10**8),
             "filter on both keys": _between("k1", 10, 30) + _between("k2", 1, 5)}[shape]
    _check(split_batches(rb, 10_000), preds, ["k1", "k2"], SUM_V)


@pytest.mark.parametrize("offset", [1, 3, 13])
def test_nullable_columns_at_bit_offsets(offset):
    rb = _table(25_000, 5, null_frac=0.15)
    _check([rb.slice(offset, 9_000), rb.slice(offset + 9_000, 11_111)], Q1, ["k1", "k2"], SUM_V + [("cv", E.AGG_COUNT, "v", T.int64)])


@pytest.mark.parametrize("key_type", [pa.int32(), pa.int16(), pa.int8()], ids=["int32", "int16", "int8"])
def test_narrow_keys(key_type):
    rb = _table(20_003, 6, null_frac=0.05, key_type=key_type)
    _check(split_batches(rb.slice(1), 8_000), Q1, ["k1", "k2"], SUM_V)
    _check([rb], [], ["k1"], SUM_V)


def test_count_of_a_column_reads_only_its_validity():
    rb = _table(20_000, 7, null_frac=0.2)
    _check(split_batches(rb, 6_000), Q1, ["k1"], [("cv", E.AGG_COUNT, "v", T.int64), ("n", E.AGG_COUNT, None, T.int64)])


WIDE = {
    "sum f64 + count": ([("s", E.AGG_SUM, "x", T.float64), ("c", E.AGG_COUNT, "x", T.int64)], (0,)),
    "sum dec + count": ([("s", E.AGG_SUM, "d", T.decimal128(27, 2)), ("c", E.AGG_COUNT, "d", T.int64)], ()),
    "min max int": ([("mn", E.AGG_MIN, "v", T.int64), ("mx", E.AGG_MAX, "v", T.int64)], ()),
    "min max f64": ([("mn", E.AGG_MIN, "x", T.float64), ("mx", E.AGG_MAX, "x", T.float64)], ()),
}


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
@pytest.mark.parametrize("shape", list(WIDE))
def test_wide_kernel_arguments(shape, null_frac):
    specs, fcols = WIDE[shape]
    rb = _table(128 * 40 + 63, 8, null_frac=null_frac, dec=True)
    _check([rb.slice(3, 2_000), rb.slice(2_003)], Q1, ["k1", "k2"], specs, float_cols=fcols)


def test_hashed_fallback_with_deferred_rows():
    """the first batch fixes a small dense range; later batches bring NULL keys and many keys outside it, so the hashed table
    fills and grows and rows are deferred and replayed by their launch-relative index"""
    rb = _table(60_000, 9)
    rng = np.random.default_rng(9)
    k1 = np.where(rng.random(60_000) < 0.5, rng.integers(100, 200_000, 60_000), rng.integers(0, 50, 60_000))
    k1[:10_000] = rng.integers(0, 50, 10_000)
    rb = rb.set_column(1, "k1", pa.array(k1, mask=rng.random(60_000) < 0.05))
    conf = native.default_conf(staging_rows=0, agg_initial_groups=256)
    _check(split_batches(rb, 10_000), Q1, ["k1", "k2"], SUM_V, conf=conf)
    _check(split_batches(rb, 10_000), Q1, ["k1"], WIDE["min max int"][0], conf=conf)


def _device_sliced(rb, torch, offset, length):
    """the columns of `rb` as device buffers, exported with Arrow offset `offset`: for an odd offset the int64 values start 8
    bytes past a 16-byte boundary; decimal128 values always do; validity starts at bit `offset`"""
    cols, keep = [], []
    for c in rb.columns:
        width = 16 if pa.types.is_decimal(c.type) else c.type.bit_width // 8
        pad = 8 if width == 16 else 0                                # decimal128: start the buffer 8 bytes past an allocation boundary
        vals = torch.tensor(np.concatenate([np.zeros(pad, np.uint8), np.frombuffer(c.buffers()[1], np.uint8)[c.offset * width:(c.offset + len(c)) * width]]), device="cuda")
        valid = None
        if c.null_count:
            valid = torch.tensor(np.packbits(c.is_valid().to_numpy(zero_copy_only=False), bitorder="little"), device="cuda")
        cols.append((vals.data_ptr() + pad, valid.data_ptr() if valid is not None else 0, len(c)))
        keep += [vals] + ([valid] if valid is not None else [])
    db = native.DeviceBatch(cols, len(rb), 0, keep)
    for i in range(db.n):
        db.children[i].offset = offset
    db.dev.array.length = length
    return db


@pytest.mark.parametrize("offset", [1, 3])
def test_device_columns_8_byte_aligned(offset):
    torch = pytest.importorskip("torch")
    rb = _table(30_000, 10, null_frac=0.1, dec=True)
    n = 128 * 150 + 31
    for specs, fcols in (([("s", E.AGG_SUM, "v", T.int64), ("cv", E.AGG_COUNT, "v", T.int64)], ()), WIDE["sum dec + count"]):
        _check([rb.slice(offset, n)], Q1, ["k1", "k2"], specs, float_cols=fcols, push=[_device_sliced(rb, torch, offset, n)])
