"""Inputs and plans shared by the WindowExec tests: the reference's KATs (tests/golden/window_kats.json), sorted random tables,
the same window as a GPU plan and as the oracle, and a brute-force restatement (every row rescans from its partition start)."""
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from blaze_b200 import exprs as E, plans as PL, types as T
from oracle import blaze_oracle as O
from oracle import window_oracle as W

KATS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "window_kats.json")))["cases"]
RANKS = {"row_number": E.ROW_NUMBER, "rank": E.RANK, "dense_rank": E.DENSE_RANK}
AGGS = {"min": E.AGG_MIN, "max": E.AGG_MAX, "sum": E.AGG_SUM, "avg": E.AGG_AVG, "count": E.AGG_COUNT}


def window_expr(name, fn, arg=None, schema=None, return_type=None):
    if fn in RANKS:
        return E.WindowExpr.rank_like(name, RANKS[fn])
    dt = schema.field(arg).dtype if hasattr(schema, "field") else next(f.dtype for f in schema if f.name == arg)
    if fn == "count":
        rt = T.int64
    elif fn in ("min", "max"):
        rt = dt
    else:
        rt = return_type or (dt if dt.is_decimal or dt.id == T.FLOAT64 else T.int64 if fn == "sum" else T.float64)
    return E.WindowExpr.agg(name, AGGS[fn], [E.Column(arg)], rt, fn != "count")


def kat_input(case):
    names = list(case["input"])
    rb = pa.RecordBatch.from_arrays([pa.array(case["input"][n], pa.int32()) for n in names], names=names)
    schema = T.Schema([T.Field(n, T.int32, False) for n in names])
    return schema, rb


def kat_window(case, schema):
    exprs = [window_expr(w[0], w[1], w[2] if len(w) > 2 else None, schema) for w in case["window_exprs"]]
    return exprs, [E.Column(c) for c in case["partition_spec"]], [(E.Column("b1"), False, True)]


def sorted_table(rb: pa.RecordBatch, keys):
    """rows sorted by `keys` (ascending, NULLs first), so that equal keys form runs as below a WindowExec"""
    t = pa.Table.from_batches([rb])
    idx = pc.sort_indices(t, sort_keys=[(k, "ascending") for k in keys], null_placement="at_start")
    return t.take(idx).combine_chunks().to_batches()[0]


def gpu_plan(schema, exprs, partition, order, group_limit=None, output_window_cols=True, batches=()):
    return PL.WindowExec(PL.MemoryExec(schema, list(batches)), exprs, partition, order, group_limit, output_window_cols)


def oracle_run(schema, exprs, partition, order, batches, group_limit=None, output_window_cols=True):
    w = W.WindowExec(exprs, partition, order, schema, group_limit, output_window_cols)
    return w.schema, w.execute([O.batch_from_arrow(b) for b in batches])


def brute_force(rb: pa.RecordBatch, fn, part, order, arg=None):
    """one window column, each row rescanned from its partition start (the semantics the processors implement, restated)"""
    n = rb.num_rows
    def keys(names):
        cols = [O.col_from_arrow(rb.column(rb.schema.get_field_index(c))) for c in names]
        return W.key_rows(cols, n)
    pk, ok = keys(part), keys(order)
    vals = rb.column(rb.schema.get_field_index(arg)).to_pylist() if arg else None
    out = []
    for i in range(n):
        s = i
        if part:
            while s > 0 and pk[s - 1] == pk[i]:
                s -= 1
        else:
            s = 0
        if fn == "row_number":
            out.append(W.wrap_i32(i - s + 1))
        elif fn in ("rank", "dense_rank"):
            if not part and not order:
                out.append(0)
                continue
            heads = [j for j in range(s, i + 1) if j == s or ok[j] != ok[j - 1]]
            out.append(W.wrap_i32(len(heads) if fn == "dense_rank" else heads[-1] - s + 1))
        else:
            seen = [v for v in vals[s:i + 1] if v is not None]
            if fn == "count":
                out.append(len(seen))
            elif not seen:
                out.append(None)
            elif fn == "sum":
                out.append(O.wrap_i64(sum(seen)) if isinstance(seen[0], int) else sum(seen))
            elif fn == "min":
                out.append(min(seen))
            else:
                out.append(max(seen))
    return out
