"""FIRST / FIRST_IGNORES_NULL in AggExec on the GPU against the row-by-row oracle (tests/first_oracle.py) or an exact Python
restatement: the reference's test_agg golden, every fixed-width value type bit for bit, Partial -> Final in every form, arrival
order across launch chunks, deferred replays, the staging ring and device-resident input, the dropDuplicates and multi-DISTINCT
plan shapes, and a fused ROLLUP."""
import decimal
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from blaze_b200.types import Field, Schema
from oracle import blaze_oracle as O
from oracle import expand_oracle as X
from helpers import *
from expand_cases import expand_for_sets, grouping_sets
import first_oracle as FO

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIRST, FIGN = E.AGG_FIRST, E.AGG_FIRST_IGNORES_NULL


def aggs(mode, specs, ins):
    """specs: (name, fn, column, return type); the Final side gets a Null-typed Placeholder for FIRST, a typed one otherwise"""
    def ch(c, fn):
        if mode == E.PARTIAL:
            return [E.Column(c)]
        return [E.placeholder() if fn in FO.FIRST_FNS else E.placeholder(ins[ins.index_of(c)].dtype)]
    return [E.AggExpr(nm, mode, PL.create_agg(fn, ch(c, fn), ins, rt)) for nm, fn, c, rt in specs]


def conf(**kw):
    return native.default_conf(**kw)


def oracle(batches, groupings, specs, ins, parts=1):
    """Partial over `parts` consecutive slices of the batches (each its own op), then one Final over the states in order"""
    ob = oracle_batches(batches)
    mid = []
    for p in range(parts):
        mid += FO.AggExec(E.HASH_AGG, groupings, aggs(E.PARTIAL, specs, ins), False, ins).execute(ob[p * len(ob) // parts:(p + 1) * len(ob) // parts])
    st = FO.AggExec(E.HASH_AGG, groupings, aggs(E.PARTIAL, specs, ins), False, ins).schema
    return FO.AggExec(E.HASH_AGG, groupings, aggs(E.FINAL, specs, ins), False, st).execute(mid)


def one_op(batches, groupings, specs, cf=None, schema=None):
    leaf = PL.MemoryExec.from_arrow(batches, schema or batches[0].schema)
    ins = leaf.schema()
    partial = PL.AggExec(PL.HashAgg, groupings, aggs(E.PARTIAL, specs, ins), False, leaf)
    final = PL.AggExec(PL.HashAgg, groupings, aggs(E.FINAL, specs, ins), False, partial)
    return PL.collect(final, cf), final.last_metrics


def two_ops(batch_groups, groupings, specs, cf=None, columnar=False):
    """one Partial op per group of batches, then one Final op over all their outputs, in order"""
    ins = T.from_arrow_schema(batch_groups[0][0].schema)
    parts, pschema = [], None
    for bg in batch_groups:
        partial = PL.AggExec(PL.HashAgg, groupings, aggs(E.PARTIAL, specs, ins), False, PL.MemoryExec.from_arrow(bg, bg[0].schema), columnar_state=columnar)
        c = conf(partial_state_columnar=1) if columnar else cf
        parts += PL.collect(partial, c)
        pschema = partial.schema()
        assert partial.last_metrics["fast_path_launches"] == 0
    final = PL.AggExec(PL.HashAgg, groupings, aggs(E.FINAL, specs, ins), False, PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(pschema)))
    return PL.collect(final, conf(partial_state_columnar=1) if columnar else cf)


def rows_of(batches, nkeys):
    """{key tuple: tuple of aggregate values}; floats as their bit patterns, so NaN payloads and -0.0 compare exactly"""
    out = {}
    for rb in batches:
        for r in range(rb.num_rows):
            row = []
            for c in rb.columns:
                v = c[r].as_py()
                if v is not None and pa.types.is_float64(c.type):
                    v = ("f64", struct.unpack("<Q", struct.pack("<d", v))[0])
                elif v is not None and pa.types.is_float32(c.type):
                    v = ("f32", struct.unpack("<I", struct.pack("<f", v))[0])
                row.append(v)
            key = tuple(row[:nkeys])
            assert key not in out, f"group {key} emitted twice"
            out[key] = tuple(row[nkeys:])
    return out


def oracle_rows(obatches, nkeys):
    return rows_of([O.batch_to_arrow(b) for b in obatches], nkeys)


# ---- the reference's golden ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch_rows", [7, 1])
def test_reference_kat_test_agg_with_first_ignores_null(batch_rows):
    g = json.load(open(os.path.join(HERE, "golden", "first_kats.json")))
    rb = rb_from_cols(list(g["input"]), [pa.array(v, pa.int32()) for v in g["input"].values()])
    specs = [("agg_expr_sum", E.AGG_SUM, "a", T.int64), ("agg_expr_avg", E.AGG_AVG, "b", T.float64), ("agg_expr_max", E.AGG_MAX, "d", T.int32),
             ("agg_expr_min", E.AGG_MIN, "e", T.int32), ("agg_expr_count", E.AGG_COUNT, "f", T.int64), ("agg_agg_firstign", FIGN, "h", T.int32)]
    got, m = one_op(split_batches(rb, batch_rows), [E.GroupingExpr("c", E.Column("c"))], specs, conf(staging_rows=0))
    assert pa.Table.from_batches(got).sort_by("c").to_pydict() == g["expected"]
    assert m["fast_path_launches"] == 0


# ---- every value type, bit for bit -------------------------------------------------------------------------------
NAN_PAYLOAD = struct.unpack("<d", struct.pack("<Q", 0x7FF8DEADBEEF1234))[0]
NEG_NAN = struct.unpack("<d", struct.pack("<Q", 0xFFF0000000000777))[0]


def typed_values(name, n, rng):
    if name == "f64":
        special = [NAN_PAYLOAD, -0.0, float("inf"), float("-inf"), NEG_NAN, 0.0, 5e-324]
        return pa.array([special[i % len(special)] if i % 3 == 0 else float(rng.normal()) for i in range(n)], pa.float64())
    if name == "f32":
        return pa.array([[-0.0, float("inf"), float("-inf"), 1.5][i % 4] if i % 3 == 0 else float(np.float32(rng.normal())) for i in range(n)], pa.float32())
    if name == "dec":
        big = 10**38 - 1
        return pa.array([decimal.Decimal([big, -big, 0, 1][i % 4] if i % 2 == 0 else int(rng.integers(-10**18, 10**18)) * 10**12 + int(rng.integers(0, 10**12))) for i in range(n)], pa.decimal128(38, 0))
    if name == "bool":
        return pa.array(rng.random(n) < 0.5, pa.bool_())
    t = {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "date": pa.date32(), "ts": pa.timestamp("us")}[name]
    info = np.iinfo({"i8": np.int8, "i16": np.int16, "i32": np.int32, "i64": np.int64, "date": np.int32, "ts": np.int64}[name])
    lo, hi = {"date": (-719162, 2932896), "ts": (-62135596800 * 10**6, 253402300799 * 10**6)}.get(name, (info.min, info.max))   # years 1..9999: Python can hold them
    raw = rng.integers(lo, hi, n, dtype=np.int64, endpoint=True)
    raw[::5] = lo
    return pa.array(raw, type=pa.int64()).cast(t) if name not in ("date", "ts") else pa.array(raw.astype(np.int32 if name == "date" else np.int64)).cast(t)


TYPES = ["i8", "i16", "i32", "i64", "date", "ts", "f32", "f64", "dec", "bool"]


@pytest.mark.parametrize("form", ["one_op", "two_ops", "columnar"])
@pytest.mark.parametrize("tname", TYPES)
def test_every_value_type_bit_exact(tname, form):
    rng = np.random.default_rng(TYPES.index(tname))
    n = 20_000
    v = typed_values(tname, n, rng)
    null = rng.random(n) < 0.4
    vals = pa.array([None if null[i] else x for i, x in enumerate(v.to_pylist())], v.type)
    k = rng.integers(0, 3000, n, dtype=np.int64)
    rb = rb_from_cols(["k", "v"], [pa.array(k), vals])
    dt = T.from_arrow_type(vals.type)
    specs = [("f", FIRST, "v", dt), ("fn", FIGN, "v", dt)]
    g = [E.GroupingExpr("k", E.Column("k"))]
    batches = split_batches(rb, 3_000)
    if form == "one_op":
        got, m = one_op(batches, g, specs)
        assert m["fast_path_launches"] == 0
    else:
        got = two_ops([batches[:3], batches[3:]], g, specs, columnar=form == "columnar")
    # exact restatement: the first row of each key, and its first valid row
    py = vals.to_pylist()
    want_f, want_n = FO.brute_force_first(list(k), py, False), FO.brute_force_first(list(k), py, True)
    exp = rows_of([pa.RecordBatch.from_arrays([pa.array(list(want_f), pa.int64()), pa.array([want_f[x] for x in want_f], vals.type),
                                               pa.array([want_n[x] for x in want_f], vals.type)], names=["k", "f", "fn"])], 1)
    assert rows_of(got, 1) == exp


# ---- Partial -> Final forms over several partial outputs, against the oracle ---------------------------------------------------
def mixed_input(n=60_000, seed=5, card=4_000):
    rng = np.random.default_rng(seed)
    return rb_from_cols(["k", "a", "b", "x", "d"],
                        [with_nulls(rng, rng.integers(0, card, n, dtype=np.int64), 0.02), with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.7),
                         with_nulls(rng, rng.integers(-100, 100, n).astype(np.int32), 0.2), with_nulls(rng, rng.normal(0, 1, n), 0.5),
                         pa.array([None if rng.random() < 0.3 else decimal.Decimal(int(x)).scaleb(-2) for x in rng.integers(-10**15, 10**15, n)], pa.decimal128(20, 2))])


MIXED_SPECS = [("fa", FIRST, "a", T.int64), ("na", FIGN, "a", T.int64), ("fb", FIRST, "b", T.int32), ("fx", FIRST, "x", T.float64),
               ("nx", FIGN, "x", T.float64), ("nd", FIGN, "d", T.decimal128(20, 2)), ("s", E.AGG_SUM, "a", T.int64), ("c", E.AGG_COUNT, "b", T.int64)]


@pytest.mark.parametrize("form", ["one_op", "two_ops", "two_ops_columnar", "three_partials"])
def test_partial_final_forms(form):
    rb = mixed_input()
    batches = split_batches(rb, 4_000)
    g = [E.GroupingExpr("k", E.Column("k"))]
    ins = T.from_arrow_schema(rb.schema)
    if form == "one_op":
        got, m = one_op(batches, g, MIXED_SPECS)
        assert m["fast_path_launches"] == 0
        parts = 1
    elif form == "three_partials":
        parts = 3
        got = two_ops([batches[p * len(batches) // 3:(p + 1) * len(batches) // 3] for p in range(3)], g, MIXED_SPECS)
    else:
        parts = 1
        got = two_ops([batches], g, MIXED_SPECS, columnar=form.endswith("columnar"))
    assert rows_of(got, 1) == oracle_rows(oracle(batches, g, MIXED_SPECS, ins, parts), 1)


@pytest.mark.skipif(os.environ.get("B200Q_NO_AGG_FUSION") is not None, reason="already without Partial/Final fusion")
def test_one_op_again_without_partial_final_fusion():
    env = dict(os.environ, B200Q_NO_AGG_FUSION="1")
    r = subprocess.run([sys.executable, "-m", "pytest", __file__, "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "partial_final_forms and one_op or rollup"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ---- arrival order under stress -----------------------------------------------------------------------------------
def test_one_group_over_device_resident_rows_takes_row_zero():
    torch = pytest.importorskip("torch")
    n = 1 << 24
    rng = np.random.default_rng(9)
    k = np.zeros(n, np.int64)
    v = rng.integers(1, 2**62, n, dtype=np.int64)
    f = rng.normal(0, 1, n)
    v[0], f[0] = -12345, NAN_PAYLOAD
    tk, tv, tf = (torch.from_numpy(x).cuda() for x in (k, v, f))
    ins = Schema([Field("k", T.int64, False), Field("v", T.int64, False), Field("f", T.float64, False)])
    specs = [("fv", FIRST, "v", T.int64), ("ff", FIRST, "f", T.float64), ("nv", FIGN, "v", T.int64)]
    g = [E.GroupingExpr("k", E.Column("k"))]
    plan = PL.AggExec(PL.HashAgg, g, aggs(E.FINAL, specs, ins), False, PL.AggExec(PL.HashAgg, g, aggs(E.PARTIAL, specs, ins), False, PL.MemoryExec(ins)))
    results = []
    for _ in range(2):
        with native.NativeOp(plan.plan_bytes(), conf()) as op:
            op.push_device(native.DeviceBatch([(tk.data_ptr(), 0, n), (tv.data_ptr(), 0, n), (tf.data_ptr(), 0, n)], n, 0, keepalive=(tk, tv, tf)))
            op.finish()
            results.append(rows_of(op.pull_all(), 1))
            assert op.metrics()["fast_path_launches"] == 0
    assert results[0] == {(0,): (-12345, ("f64", 0x7FF8DEADBEEF1234), -12345)}
    assert results[1] == results[0]


def test_first_rows_in_later_launch_chunks_and_deferred_replays():
    """700 k unique keys, beyond the load limit of the first table (2^19 groups): the table grows and the deferred rows of the chunk
    that hit the limit are replayed; every key appears again in a later chunk, and a key whose first occurrence is NULL keeps that
    NULL under FIRST"""
    rng = np.random.default_rng(13)
    n_keys = 700_000
    first = rng.permutation(n_keys).astype(np.int64)
    again = rng.permutation(n_keys).astype(np.int64)
    k = np.concatenate([first, again])
    v = np.arange(2 * n_keys, dtype=np.int64)
    null = np.zeros(2 * n_keys, bool)
    null[:n_keys] = rng.random(n_keys) < 0.3
    rb = rb_from_cols(["k", "v"], [pa.array(k), pa.array(v, mask=null)])
    specs = [("f", FIRST, "v", T.int64), ("fn", FIGN, "v", T.int64)]
    g = [E.GroupingExpr("k", E.Column("k"))]
    cf = conf(agg_initial_groups=1024, max_launch_rows=1 << 16, staging_rows=0)
    got, m = one_op([rb], g, specs, cf)
    assert m["table_grow_count"] >= 1
    py = [None if null[i] else int(v[i]) for i in range(2 * n_keys)]
    wf, wn = FO.brute_force_first(list(k), py, False), FO.brute_force_first(list(k), py, True)
    assert rows_of(got, 1) == {(int(key),): (wf[key], wn[key]) for key in wf}


def test_pageable_batches_through_the_staging_ring():
    rb = mixed_input(n=120_000, seed=17, card=30_000)
    batches = split_batches(rb, 10_000)
    g = [E.GroupingExpr("k", E.Column("k"))]
    got, _ = one_op(batches, g, MIXED_SPECS, conf(staging_rows=65_536))
    assert rows_of(got, 1) == oracle_rows(oracle(batches, g, MIXED_SPECS, T.from_arrow_schema(rb.schema)), 1)


# ---- no grouping --------------------------------------------------------------------------------------------------
def test_global_first_empty_and_all_null():
    specs = [("f", FIRST, "v", T.int64), ("fn", FIGN, "v", T.int64)]
    schema = pa.schema([("v", pa.int64())])
    empty = pa.RecordBatch.from_arrays([pa.array([], pa.int64())], schema=schema)
    nulls = pa.RecordBatch.from_arrays([pa.array([None] * 5, pa.int64())], schema=schema)
    for batches, state in (([empty], b"\x00\x00\x00"), ([nulls], b"\x00\x02\x00")):
        got, _ = one_op(batches, [], specs)
        assert pa.Table.from_batches(got).to_pydict() == {"f": [None], "fn": [None]}
        partial = PL.AggExec(PL.HashAgg, [], aggs(E.PARTIAL, specs, T.from_arrow_schema(schema)), False, PL.MemoryExec.from_arrow(batches, schema))
        assert pa.Table.from_batches(PL.collect(partial)).column(0).to_pylist() == [state]      # value NULL; FIRST's flag set iff a row came


# ---- plan shapes ----------------------------------------------------------------------------------------------------
def test_drop_duplicates_shape():
    """Dataset.dropDuplicates(k): Aggregate(k, first(c, ignoreNulls = false) for 12 columns of mixed types)"""
    rng = np.random.default_rng(23)
    n = 80_000
    names = [f"c{i}" for i in range(12)]
    mk = [lambda: rng.integers(-10**12, 10**12, n, dtype=np.int64), lambda: rng.integers(-100, 100, n).astype(np.int32),
          lambda: rng.normal(0, 1, n), lambda: rng.integers(-100, 100, n).astype(np.int8), lambda: rng.random(n) < 0.5,
          lambda: rng.normal(0, 1, n).astype(np.float32)]
    cols = [with_nulls(rng, mk[i % len(mk)](), 0.15) for i in range(10)]
    cols.append(pa.array(rng.integers(0, 20_000, n).astype(np.int32), pa.int32()).cast(pa.date32()))
    cols.append(pa.array([None if rng.random() < 0.2 else decimal.Decimal(int(x)).scaleb(-4) for x in rng.integers(-10**17, 10**17, n)], pa.decimal128(24, 4)))
    rb = rb_from_cols(["k"] + names, [pa.array(rng.integers(0, 15_000, n, dtype=np.int64))] + cols)
    ins = T.from_arrow_schema(rb.schema)
    specs = [(f"first_{c}", FIRST, c, ins[ins.index_of(c)].dtype) for c in names]
    g = [E.GroupingExpr("k", E.Column("k"))]
    batches = split_batches(rb, 7_000)
    for got in (one_op(batches, g, specs)[0], two_ops([batches], g, specs), two_ops([batches], g, specs, columnar=True)):
        assert rows_of(got, 1) == oracle_rows(oracle(batches, g, specs, ins), 1)


def test_multi_distinct_rewrite_end_to_end():
    """COUNT(DISTINCT a), COUNT(DISTINCT b), SUM(c) GROUP BY k as Spark's RewriteDistinctAggregates plans it:
    Expand(gid) -> Agg(Partial) -> Agg(Final) over (k, a, b, gid) -> Agg(Partial) [COUNT(If(gid=1, a)), COUNT(If(gid=2, b)),
    FIRST_IGNORES_NULL(If(gid=0, sum_c))] -> Agg(Final), checked against a direct computation"""
    rng = np.random.default_rng(29)
    n = 50_000
    k = rng.integers(0, 300, n, dtype=np.int64)
    a = rng.integers(0, 40, n).astype(np.int32)
    b = rng.integers(-25, 25, n, dtype=np.int64)
    c = rng.integers(-10**9, 10**9, n, dtype=np.int64)
    an, bn, cn = rng.random(n) < 0.1, rng.random(n) < 0.1, rng.random(n) < 0.1
    rb = rb_from_cols(["k", "a", "b", "c"], [pa.array(k), pa.array(a, mask=an), pa.array(b, mask=bn), pa.array(c, mask=cn)])
    batches = split_batches(rb, 8_000)
    fields = [Field("k", T.int64, False), Field("a", T.int32, True), Field("b", T.int64, True), Field("gid", T.int32, False), Field("c", T.int64, True)]
    n32, n64 = E.Literal(None, T.int32), E.Literal(None, T.int64)
    projs = [[E.Column("k"), n32, n64, E.Literal(0, T.int32), E.Column("c")], [E.Column("k"), E.Column("a"), n64, E.Literal(1, T.int32), n64],
             [E.Column("k"), n32, E.Column("b"), E.Literal(2, T.int32), n64]]
    es = Schema(fields)
    g1 = [E.GroupingExpr(x, E.Column(x)) for x in ("k", "a", "b", "gid")]
    s1 = [("sum_c", E.AGG_SUM, "c", T.int64)]
    p1 = PL.AggExec(PL.HashAgg, g1, aggs(E.PARTIAL, s1, es), False, PL.ExpandExec(es, projs, PL.MemoryExec.from_arrow(batches, rb.schema)))
    f1 = PL.AggExec(PL.HashAgg, g1, aggs(E.FINAL, s1, es), False, p1)
    lvl1 = PL.collect(f1)
    ls = T.from_arrow_schema(lvl1[0].schema)
    gid = E.Column("gid")
    when = lambda val, col, dt: E.Case(None, [(E.BinaryExpr(gid, "Eq", E.Literal(val, T.int32)), E.Column(col))], E.Literal(None, dt))
    args = [("cnt_a", E.AGG_COUNT, when(1, "a", T.int32), T.int64), ("cnt_b", E.AGG_COUNT, when(2, "b", T.int64), T.int64),
            ("sum_c", FIGN, when(0, "sum_c", T.int64), T.int64)]
    g2 = [E.GroupingExpr("k", E.Column("k"))]
    p2 = PL.AggExec(PL.HashAgg, g2, [E.AggExpr(nm, E.PARTIAL, PL.create_agg(fn, [ex], ls, rt)) for nm, fn, ex, rt in args], False,
                    PL.MemoryExec.from_arrow(lvl1, lvl1[0].schema))
    f2 = PL.AggExec(PL.HashAgg, g2, [E.AggExpr(nm, E.FINAL, PL.create_agg(fn, [E.placeholder() if fn == FIGN else E.placeholder(T.int64)], ls, rt))
                                      for nm, fn, ex, rt in args], False, p2)
    got = pa.Table.from_batches(PL.collect(f2)).sort_by("k").to_pydict()
    exp = {"k": [], "cnt_a": [], "cnt_b": [], "sum_c": []}
    for key in sorted(set(k.tolist())):
        sel = k == key
        exp["k"].append(key)
        exp["cnt_a"].append(len(set(a[sel & ~an].tolist())))
        exp["cnt_b"].append(len(set(b[sel & ~bn].tolist())))
        cs = c[sel & ~cn]
        exp["sum_c"].append(int(((int(cs.sum()) + 2**63) % 2**64) - 2**63) if len(cs) else None)
    assert got == exp


def test_fused_rollup_with_grouping_id():
    rng = np.random.default_rng(31)
    n = 40_000
    rb = rb_from_cols(["k1", "k2", "v", "x"], [pa.array(rng.integers(0, 30, n, dtype=np.int64)), with_nulls(rng, rng.integers(0, 50, n).astype(np.int32), 0.1),
                                               with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.6), with_nulls(rng, rng.normal(0, 1, n), 0.3)])
    ins = T.from_arrow_schema(rb.schema)
    es, projs = expand_for_sets(ins, ["k1", "k2"], ["v", "x"], grouping_sets("rollup", 2))
    g = [E.GroupingExpr(x, E.Column(x)) for x in ("k1", "k2", "spark_grouping_id")]
    specs = [("nv", FIGN, "v", T.int64), ("fx", FIRST, "x", T.float64), ("nx", FIGN, "x", T.float64), ("s", E.AGG_SUM, "v", T.int64)]
    batches = split_batches(rb, 6_000)
    partial = PL.AggExec(PL.HashAgg, g, aggs(E.PARTIAL, specs, es), False, PL.ExpandExec(es, projs, PL.MemoryExec.from_arrow(batches, rb.schema)))
    got = PL.collect(PL.AggExec(PL.HashAgg, g, aggs(E.FINAL, specs, es), False, partial))
    op = FO.AggExec(E.HASH_AGG, g, aggs(E.PARTIAL, specs, es), False, es)
    of = FO.AggExec(E.HASH_AGG, g, aggs(E.FINAL, specs, es), False, op.schema)
    exp = of.execute(op.execute(X.ExpandExec(es, projs, ins).execute(oracle_batches(batches))))
    assert rows_of(got, 3) == oracle_rows(exp, 3)
