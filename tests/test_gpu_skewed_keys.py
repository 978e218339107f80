"""Skewed keys: the skew probe on the first batch selects the CTA-private hot-key cache kernel
(b200q_conf.agg_hot_key_cache, on by default)."""
import os

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
from oracle import blaze_oracle as O
from helpers import *

pytestmark = pytest.mark.gpu


def zipf_keys(rng, n, nkeys, s=1.1):
    u = rng.random(n)
    ranks = np.clip(np.floor((u * (nkeys ** (1 - s) - 1) + 1) ** (1 / (1 - s))).astype(np.int64), 1, nkeys) - 1
    return (ranks * 2654435761) % nkeys


@pytest.mark.parametrize("shape", ["sum+count*", "sum+count(v) nullable schema", "two keys + filter", "sum only"])
def test_hot_key_cache_on_skewed_keys(shape):
    n = 600_000
    rng = np.random.default_rng(91)
    k = zipf_keys(rng, n, 50_000).astype(np.int64) - 7
    k[400_000:] += rng.integers(0, 200_000, n - 400_000)                  # later batches leave the dense range of the first one
    v = rng.integers(-2**40, 2**40, n, dtype=np.int64)
    f = rng.integers(0, 100, n, dtype=np.int64)
    k2 = rng.integers(0, 5, n, dtype=np.int64)
    nullable = shape == "sum+count(v) nullable schema"
    schema = pa.schema([pa.field(c, pa.int64(), nullable=nullable) for c in ("k", "k2", "f", "v")])
    rb = pa.RecordBatch.from_arrays([pa.array(k), pa.array(k2), pa.array(f), pa.array(v)], schema=schema)
    batches = split_batches(rb, 150_000)
    leaf = PL.MemoryExec.from_arrow(batches, rb.schema)
    ins = leaf.schema()
    groupings = [E.GroupingExpr("k", E.Column("k"))] + ([E.GroupingExpr("k2", E.Column("k2"))] if shape.startswith("two") else [])
    aggs = [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], ins, T.int64))]
    if shape == "sum+count*":
        aggs.append(E.AggExpr("n", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Literal(1, T.int64)], ins, T.int64)))
    elif shape != "sum only":
        aggs.append(E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Column("v")], ins, T.int64)))
    preds = [E.BinaryExpr(E.Column("f"), "Lt", E.Literal(70, T.int64))] if shape.startswith("two") else []
    child = PL.FilterExec(preds, leaf) if preds else leaf
    plan = PL.AggExec(PL.HashAgg, groupings, aggs, False, child)
    got = PL.collect(plan, native.default_conf(staging_rows=0, agg_hot_key_cache=1))
    ob = oracle_batches(batches)
    exp = O.AggExec(E.HASH_AGG, groupings, aggs, False, ins).execute(O.FilterExec(preds, ins).execute(ob) if preds else ob)
    assert_multiset_equal(got, exp)
    assert plan.last_metrics["fast_path_launches"] > 0
