"""The dense-table decision of AggExec, taken on the first batch from the key ranges of (a sample of) its rows: every key's
range is padded by r/8 + min(64, r/2 + 1) on each side, the table has prod(padded ranges) entries, and it is used only
while that is <= 8 x max(non-null rows, agg_initial_groups, 65536) entries, <= 2^26 entries and, when
agg_max_table_bytes > 0, within that many bytes.  Outside those bounds the op stays on the hash table.

The wide tile kernel (SUM over f64) counts its launches in fast_path_launches and the generic VM kernel counts none,
so for those plans the test sees which side of the boundary the decision fell on.  Every result is checked against the
oracle."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
from oracle import blaze_oracle as O
from helpers import *

pytestmark = pytest.mark.gpu

INITIAL_GROUPS = 1024        # below the 65536 floor, so the entry budget is 8 x max(rows, 65536)


def padded_span(r):
    return r + 2 * (r // 8 + min(64, r // 2 + 1))


def entry_budget(rows):
    return 8 * max(rows, INITIAL_GROUPS, 1 << 16)


def widest_dense_range(rows):
    """the largest key range r whose padded span still fits the entry budget of `rows` rows"""
    r = entry_budget(rows)
    while padded_span(r) > entry_budget(rows):
        r -= 1
    return r


def _keys(rng, n, r, distinct=None):
    """int64 keys spanning exactly [0, r): both ends present; `distinct` limits the number of different keys"""
    k = rng.integers(0, r, n, dtype=np.int64) if distinct is None else rng.choice(rng.integers(0, r, distinct, dtype=np.int64), n)
    k[0], k[1] = 0, r - 1
    return k


def _values(rng, n):
    """f64 integers: every summation order gives the same sum"""
    return rng.integers(0, 1000, n).astype(np.float64)


def _run(cols, aggs, conf, float_cols=()):
    """AggExec(Partial) -> AggExec(Final) grouped by every `k*` column, one input batch; returns fast_path_launches"""
    rb = pa.RecordBatch.from_arrays([pa.array(v) for v in cols.values()], names=list(cols))
    leaf = PL.MemoryExec.from_arrow([rb], rb.schema)
    ins = leaf.schema()
    g = [E.GroupingExpr(c, E.Column(c)) for c in cols if c.startswith("k")]
    mk = lambda mode, src: [E.AggExpr(nm, mode, PL.create_agg(fn, [E.Column(col)] if mode == E.PARTIAL else [E.placeholder(rt)], src, rt))
                            for nm, fn, col, rt in aggs]
    partial = PL.AggExec(PL.HashAgg, g, mk(E.PARTIAL, ins), False, leaf)
    final = PL.AggExec(PL.HashAgg, g, mk(E.FINAL, partial.schema()), False, partial)
    got = PL.collect(final, conf)
    op = O.AggExec(E.HASH_AGG, g, mk(E.PARTIAL, ins), False, ins)
    of = O.AggExec(E.HASH_AGG, g, mk(E.FINAL, op.schema), False, op.schema)
    assert_multiset_equal(got, of.execute(op.execute(oracle_batches([rb]))), tuple(len(g) + c for c in float_cols))
    return final.last_metrics["fast_path_launches"]


SUM_F64 = [("s", E.AGG_SUM, "x", T.float64)]


def _conf(**kw):
    return native.default_conf(staging_rows=0, agg_initial_groups=INITIAL_GROUPS, **kw)


@pytest.mark.parametrize("outside", [False, True], ids=["inside", "outside"])
def test_entry_budget(outside):
    n = 100_000
    r = widest_dense_range(n) + (1 if outside else 0)
    assert (padded_span(r) > entry_budget(n)) == outside
    rng = np.random.default_rng(1 + outside)
    launches = _run({"k": _keys(rng, n, r), "x": _values(rng, n)}, SUM_F64, _conf(), (0,))
    assert (launches == 0) == outside, f"r = {r}: padded span {padded_span(r)} against a budget of {entry_budget(n)} entries"


@pytest.mark.parametrize("admits_dense", [False, True], ids=["hash only", "dense too"])
def test_byte_budget(admits_dense):
    n = 1 << 19
    r = 2_400_000
    entries = padded_span(r)
    assert entries <= entry_budget(n) and entries <= 1 << 26
    # hash table: max(2^20, 3 x 1024) slots of {header, key} + at most 2 accumulator words; dense table: >= 2 words per entry
    hash_bytes = (1 << 20) * (2 + 2) * 8
    dense_bytes_min, dense_bytes_max = entries * 2 * 8, entries * 4 * 8
    assert dense_bytes_min > hash_bytes
    budget = dense_bytes_max if admits_dense else hash_bytes
    rng = np.random.default_rng(3)
    cols = {"k": _keys(rng, n, r, distinct=1000), "x": _values(rng, n)}     # few groups: the hash table never grows
    launches = _run(cols, SUM_F64, _conf(agg_max_table_bytes=budget), (0,))
    assert (launches > 0) == admits_dense


@pytest.mark.parametrize("r0, r1, dense", [(500, 100, True), (1000, 1000, False)])
def test_two_keys(r0, r1, dense):
    """both keys' ranges come back together; the entry count is the product of the padded spans"""
    n = 100_000
    assert (padded_span(r0) * padded_span(r1) <= entry_budget(n)) == dense
    rng = np.random.default_rng(r0 + r1)
    cols = {"k0": _keys(rng, n, r0), "k1": _keys(rng, n, r1), "x": _values(rng, n)}
    launches = _run(cols, SUM_F64, _conf(), (0,))
    assert (launches > 0) == dense


@pytest.mark.parametrize("outside", [False, True], ids=["inside", "outside"])
@pytest.mark.parametrize("hot_key_cache", [0, 1])
def test_fast_path_at_the_entry_budget(outside, hot_key_cache):
    """SUM / COUNT over int64 take the fast kernels on both sides of the boundary (dense table inside, hash table outside);
    fast_path_launches counts both, so only the results are checked here"""
    n = 100_000
    r = widest_dense_range(n) + (1 if outside else 0)
    rng = np.random.default_rng(5 + outside)
    v = rng.integers(-10**6, 10**6, n, dtype=np.int64)
    _run({"k": _keys(rng, n, r), "v": v}, [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, "v", T.int64)], _conf(agg_hot_key_cache=hot_key_cache))
