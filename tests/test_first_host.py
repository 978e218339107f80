"""FIRST / FIRST_IGNORES_NULL without a GPU: decode and explain through b200q_plan_explain, the oracle against the reference's
test_agg golden and against a brute-force restatement, and the frozen state bytes."""
import json
import os

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from blaze_b200.types import Field, Schema
from oracle import blaze_oracle as O
import first_oracle as FO

HERE = os.path.dirname(os.path.abspath(__file__))
S = Schema([Field("k", T.int64, True), Field("i", T.int32, True), Field("d", T.decimal128(20, 3), True), Field("b", T.bool_, True),
            Field("s", T.utf8, True), Field("f", T.float64, False), Field("t", T.timestamp_us, True)])


def first_aggs(mode, specs, ins):
    return [E.AggExpr(name, mode, PL.create_agg(fn, ch, ins, rt)) for name, fn, ch, rt in specs]


# ---- decode / explain -------------------------------------------------------------------------------------------
def test_explain_types_and_nullability():
    leaf = PL.MemoryExec(S)
    aggs = first_aggs(E.PARTIAL, [("fi", E.AGG_FIRST, [E.Column("i")], T.int32), ("fd", E.AGG_FIRST_IGNORES_NULL, [E.Column("d")], T.decimal128(20, 3)),
                                  ("fb", E.AGG_FIRST, [E.Column("b")], T.bool_), ("ff", E.AGG_FIRST, [E.Column("f")], T.float64)], S)
    txt = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], aggs, False, leaf).explain()
    assert "First(i@1):int32/Partial AS fi" in txt and "FirstIgnoresNull(d@2):decimal128(20,3)/Partial AS fd" in txt
    assert "First(b@3):bool/Partial AS fb" in txt and "First(f@5):float64/Partial AS ff" in txt
    final_in = Schema([Field("k", T.int64, True), Field(E.AGG_BUF_COLUMN_NAME, T.binary, False)])
    fin = first_aggs(E.FINAL, [("fi", E.AGG_FIRST, [E.placeholder()], T.int32), ("ft", E.AGG_FIRST_IGNORES_NULL, [E.placeholder()], T.timestamp_us),
                               ("ff", E.AGG_FIRST, [E.placeholder()], T.float64)], final_in)
    plan = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], fin, False, PL.MemoryExec(final_in))
    txt = plan.explain()
    # a Null-typed Placeholder on the merge side: the type comes from return_type; FIRST is always nullable (first.rs)
    assert "First(Placeholder()):int32/Final AS fi" in txt and "FirstIgnoresNull(Placeholder()):timestamp[us]/Final AS ft" in txt
    assert "schema=[k:int64?, fi:int32?, ft:timestamp[us]?, ff:float64?]" in txt
    assert [(f.name, f.dtype, f.nullable) for f in plan.schema()][1:] == [("fi", T.int32, True), ("ft", T.timestamp_us, True), ("ff", T.float64, True)]


def test_columnar_state_fields():
    leaf = PL.MemoryExec(S)
    aggs = first_aggs(E.PARTIAL, [("fi", E.AGG_FIRST, [E.Column("i")], T.int32), ("fn", E.AGG_FIRST_IGNORES_NULL, [E.Column("t")], T.timestamp_us)], S)
    p = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], aggs, False, leaf, columnar_state=True)
    assert [(f.name, f.dtype, f.nullable) for f in p.schema()] == [("k", T.int64, True), ("fi", T.int32, True), ("fi#flag", T.int8, False),
                                                                   ("fn", T.timestamp_us, True)]


@pytest.mark.parametrize("fn", [E.AGG_FIRST, E.AGG_FIRST_IGNORES_NULL])
def test_utf8_first_is_refused_with_a_message(fn):
    with pytest.raises(native.NativeError) as ei:
        PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], first_aggs(E.PARTIAL, [("x", fn, [E.Column("s")], T.utf8)], S), False, PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED
    assert ("FIRST_IGNORES_NULL" if fn == E.AGG_FIRST_IGNORES_NULL else "FIRST") in str(ei.value) and "utf8" in str(ei.value).lower()


@pytest.mark.parametrize("fn", [5, 6, 9])
def test_other_functions_stay_refused(fn):
    with pytest.raises(native.NativeError) as ei:
        PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], first_aggs(E.PARTIAL, [("x", fn, [E.Column("i")], T.int32)], S), False, PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED and f"#{fn}" in str(ei.value)


# ---- oracle -------------------------------------------------------------------------------------------------------
def final_specs(specs, ins):
    """the Final side: FIRST gets a Null-typed Placeholder (its type comes from return_type), the others a typed one"""
    return [(n, fn, [E.placeholder() if fn in FO.FIRST_FNS else E.placeholder(ch[0].data_type(ins))], rt) for n, fn, ch, rt in specs]


def run_oracle(batches, group_cols, specs, ins):
    groupings = [E.GroupingExpr(c, E.Column(c)) for c in group_cols]
    op = FO.AggExec(E.HASH_AGG, groupings, first_aggs(E.PARTIAL, specs, ins), False, ins)
    mid = op.execute(batches)
    fspecs = final_specs(specs, ins)
    of = FO.AggExec(E.HASH_AGG, groupings, first_aggs(E.FINAL, fspecs, op.schema), False, op.schema)
    return mid, of.execute(mid)


def test_oracle_reference_golden():
    g = json.load(open(os.path.join(HERE, "golden", "first_kats.json")))
    cols = g["input"]
    rb = pa.RecordBatch.from_arrays([pa.array(v, pa.int32()) for v in cols.values()], names=list(cols))
    ins = Schema([Field(c, T.int32, True) for c in cols])
    specs = [("agg_expr_sum", E.AGG_SUM, [E.Column("a")], T.int64), ("agg_expr_avg", E.AGG_AVG, [E.Column("b")], T.float64),
             ("agg_expr_max", E.AGG_MAX, [E.Column("d")], T.int32), ("agg_expr_min", E.AGG_MIN, [E.Column("e")], T.int32),
             ("agg_expr_count", E.AGG_COUNT, [E.Column("f")], T.int64), ("agg_agg_firstign", E.AGG_FIRST_IGNORES_NULL, [E.Column("h")], T.int32)]
    for rows in (7, 1):
        batches = [O.batch_from_arrow(rb.slice(i, rows)) for i in range(0, 7, rows)]
        _, out = run_oracle(batches, ["c"], specs, ins)
        t = pa.Table.from_batches([O.batch_to_arrow(b) for b in out]).sort_by("c").to_pydict()
        assert t == g["expected"]


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("batch_rows", [1, 7, 64, 1000])
def test_oracle_vs_brute_force(seed, batch_rows):
    rng = np.random.default_rng(seed)
    n = 600
    k = rng.integers(0, 40, n)
    v = rng.integers(-1000, 1000, n)
    null = rng.random(n) < (0.85 if seed == 2 else 0.3)           # NULL-heavy on one seed
    if seed == 3:
        null[:300] = True                                             # many groups see their first valid value in a later batch
    ins = Schema([Field("k", T.int64, False), Field("v", T.int64, True)])
    rb = pa.RecordBatch.from_arrays([pa.array(k), pa.array(v, mask=null)], names=["k", "v"])
    batches = [O.batch_from_arrow(rb.slice(i, batch_rows)) for i in range(0, n, batch_rows)]
    specs = [("f", E.AGG_FIRST, [E.Column("v")], T.int64), ("fn", E.AGG_FIRST_IGNORES_NULL, [E.Column("v")], T.int64)]
    mid, out = run_oracle(batches, ["k"], specs, ins)
    vals = [None if null[i] else int(v[i]) for i in range(n)]
    want_f, want_n = FO.brute_force_first(list(k), vals, False), FO.brute_force_first(list(k), vals, True)
    got = {}
    for b in out:
        for r in range(b.num_rows):
            got[int(b.cols[0].values[r])] = (FO.np_values(b.cols[1])[r], FO.np_values(b.cols[2])[r])
    assert got == {int(key): (want_f[key], want_n[key]) for key in want_f}
    # merge side: the partial states, split into several inputs and merged in order, give the same result
    for parts in (2, 5):
        groupings = [E.GroupingExpr("k", E.Column("k"))]
        states = []
        for p in range(parts):
            sub = batches[p * len(batches) // parts:(p + 1) * len(batches) // parts]
            states += FO.AggExec(E.HASH_AGG, groupings, first_aggs(E.PARTIAL, specs, ins), False, ins).execute(sub)
        st_schema = states[0].schema
        merged = FO.AggExec(E.HASH_AGG, groupings, first_aggs(E.FINAL, final_specs(specs, ins), st_schema),
                            False, st_schema).execute(states)
        got2 = {}
        for b in merged:
            for r in range(b.num_rows):
                got2[int(b.cols[0].values[r])] = (FO.np_values(b.cols[1])[r], FO.np_values(b.cols[2])[r])
        assert got2 == got


def test_no_grouping_empty_and_all_null():
    ins = Schema([Field("v", T.int64, True)])
    specs = [("f", E.AGG_FIRST, [E.Column("v")], T.int64), ("fn", E.AGG_FIRST_IGNORES_NULL, [E.Column("v")], T.int64)]
    op = FO.AggExec(E.HASH_AGG, [], first_aggs(E.PARTIAL, specs, ins), False, ins)
    assert op.execute([])[0].cols[0].values[0] == b"\x00\x00" + b"\x00"                 # value NULL, flag unset; FIRST_IGNORES_NULL NULL
    rb = pa.RecordBatch.from_arrays([pa.array([None, None], pa.int64())], names=["v"])
    assert op.execute([O.batch_from_arrow(rb)])[0].cols[0].values[0] == b"\x00\x02" + b"\x00"   # all NULL: value NULL with the flag set


# ---- frozen bytes -------------------------------------------------------------------------------------------------
def test_frozen_layout_byte_for_byte():
    assert FO.freeze_first(T.int32, None) == b"\x00\x02"                                 # value NULL, flag set
    assert FO.freeze_first(T.int32, None, flag=False) == b"\x00\x00"
    assert FO.freeze_first(T.int32, -2) == b"\x01" + (-2).to_bytes(4, "little", signed=True) + b"\x02"
    assert FO.freeze_first(T.int8, 5) == b"\x01\x05\x02"
    assert FO.freeze_first(T.decimal128(38, 0), -(10**38 - 1)) == b"\x01" + (-(10**38 - 1) % 2**128).to_bytes(16, "little") + b"\x02"
    assert FO.freeze_first(T.bool_, True) == b"\x02\x02" and FO.freeze_first(T.bool_, False) == b"\x01\x02"
    assert FO.freeze_first(T.float64, -0.0) == b"\x01" + bytes(7) + b"\x80\x02"


@pytest.mark.parametrize("dt,vals", [(T.int64, [3, None, -(2**63)]), (T.bool_, [True, None, False]), (T.float32, [1.5, None, -0.0]),
                                     (T.decimal128(38, 0), [10**38 - 1, None, -(10**38 - 1)]), (T.date32, [-1, None, 19000])])
def test_binary_round_trip(dt, vals):
    ins = Schema([Field("k", T.int64, False), Field("v", dt, True)])
    arr = pa.array([None if x is None else (__import__("decimal").Decimal(x) if dt.is_decimal else x) for x in vals], type=T.to_arrow_type(dt))
    rb = pa.RecordBatch.from_arrays([pa.array([0, 1, 2], pa.int64()), arr], names=["k", "v"])
    specs = [("f", E.AGG_FIRST, [E.Column("v")], dt), ("fn", E.AGG_FIRST_IGNORES_NULL, [E.Column("v")], dt)]
    mid, out = run_oracle([O.batch_from_arrow(rb)], ["k"], specs, ins)
    st = {int(b.cols[0].values[r]): b.cols[1].values[r] for b in mid for r in range(b.num_rows)}
    assert st[1] == b"\x00\x02\x00"                                                    # FIRST: NULL value, flag set; FIRST_IGNORES_NULL: NULL
    res = {int(b.cols[0].values[r]): (FO.np_values(b.cols[1])[r], FO.np_values(b.cols[2])[r]) for b in out for r in range(b.num_rows)}
    for key, v in enumerate(vals):
        got_f, got_n = res[key]
        if dt.is_float and v == 0.0:
            assert np.signbit(got_f) and np.signbit(got_n)
        assert got_f == v and got_n == v
