"""Every HashAgg kernel path against the exact reference of tests/exact_agg.py, on groups built around the numeric edges of
f64, f32, decimal128 and int64 aggregates: -0.0 sums, IEEE specials, subnormals, dyadic sums that are exact in any order,
ill-conditioned sums (checked against a proven error bound), decimal128 carries and i128 wrapping, int64 wrapping and
extremes, and keys at the ends of the int64 range.  Each group is compared on its own: exact results bit for bit, NaN by
NaN-ness, inexact f64 sums inside their interval, keys exactly."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
from oracle import blaze_oracle as O
from expand_cases import expand_for_sets, grouping_sets
import exact_agg as X
from exact_agg import SHAPES, family

pytestmark = pytest.mark.gpu

F64, I64 = T.float64, T.int64


def aggs(mode, specs, ins):
    ch = lambda col, rt: [E.Column(col) if col else E.Literal(1, I64)] if mode == E.PARTIAL else [E.placeholder(ins[ins.index_of(col)].dtype if col else I64)]
    return [E.AggExpr(nm, mode, PL.create_agg(fn, ch(col, rt), ins, rt)) for nm, fn, col, rt in specs]


def conf(**kw):
    return native.default_conf(staging_rows=0, **kw)


def got_groups(batches, nkeys):
    """{key tuple: [values]} of the engine's output; floats as Python floats (f32 as np.float32), decimals unscaled"""
    out = {}
    for rb in batches:
        b = O.batch_from_arrow(rb)
        for r in range(b.num_rows):
            row = []
            for c in b.cols:
                if not c.valid[r]:
                    row.append(None)
                elif c.dtype.id == T.FLOAT32:
                    row.append(np.float32(c.values[r]))
                elif c.dtype.id == T.FLOAT64:
                    row.append(float(c.values[r]))
                else:
                    row.append(int(c.values[r]))
            key = tuple(row[:nkeys])
            assert key not in out, f"group {key} emitted twice"
            out[key] = row[nkeys:]
    return out


def assert_groups(got, exp, specs, kinds=None):
    assert got.keys() == exp.keys(), f"group keys differ: {len(got.keys() - exp.keys())} extra, {len(exp.keys() - got.keys())} missing, " \
                                     f"e.g. extra {sorted(got.keys() - exp.keys(), key=repr)[:3]} missing {sorted(exp.keys() - got.keys(), key=repr)[:3]}"
    bad = []
    for k, ev in exp.items():
        for (nm, *_), e, g in zip(specs, ev, got[k]):
            if not X.matches(e, g):
                bad.append((k, (kinds or {}).get(k[0] if k else None), nm, e, g))
    assert not bad, f"{len(bad)} aggregates differ from the exact reference, e.g. " + "; ".join(f"group {k} ({kd}) {nm}: expected {e!r}, got {g!r}" for k, kd, nm, e, g in bad[:6])


def expected(tab, specs, grouped=True):
    keys = [(k,) if grouped else () for k in tab.keys]
    return X.expected_groups(keys, tab.cols, specs, tab.types)


def run_two_ops(leaf, groupings, specs, cf, columnar=False):
    partial = PL.AggExec(PL.HashAgg, groupings, aggs(E.PARTIAL, specs, leaf.schema()), False, leaf, columnar_state=columnar)
    parts = PL.collect(partial, cf)
    mid = PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(partial.schema()))
    return PL.collect(PL.AggExec(PL.HashAgg, groupings, aggs(E.FINAL, specs, leaf.schema()), False, mid), cf)


def run_one_op(leaf, groupings, specs, cf, columnar=False):
    partial = PL.AggExec(PL.HashAgg, groupings, aggs(E.PARTIAL, specs, leaf.schema()), False, leaf, columnar_state=columnar)
    final = PL.AggExec(PL.HashAgg, groupings, aggs(E.FINAL, specs, leaf.schema()), False, partial)
    return PL.collect(final, cf), final.last_metrics


PATHS = ["default", "fast_hash", "generic", "two_stage", "columnar", "rollup", "no_grouping"]


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_numeric_edges(shape, path):
    sh = SHAPES[shape]
    tab = family(sh.family)
    specs = sh.specs
    leaf = PL.MemoryExec.from_arrow(tab.batches, tab.schema)
    g = [E.GroupingExpr("k", E.Column("k"))]
    if path == "default":
        got, m = run_one_op(leaf, g, specs, conf())
        assert (m["fast_path_launches"] > 0) == sh.fast, "the shape must take the specialised kernels exactly when they cover it"
    elif path == "fast_hash":
        got, _ = run_one_op(leaf, g, specs, conf(agg_dense_keys=0))
    elif path == "generic":
        got, m = run_one_op(leaf, g, specs, conf(force_generic_kernels=1))
        assert m["fast_path_launches"] == 0
    elif path == "two_stage":
        got = run_two_ops(leaf, g, specs, conf())
    elif path == "columnar":
        cf = conf(); cf.partial_state_columnar = 1
        got, _ = run_one_op(leaf, g, specs, cf, columnar=True)
    elif path == "rollup":
        ins = leaf.schema()
        carried = sorted({c for _, _, c, _ in specs if c})
        eschema, projs = expand_for_sets(ins, ["k"], carried, grouping_sets("rollup", 1))
        gs = [E.GroupingExpr("k", E.Column("k")), E.GroupingExpr("spark_grouping_id", E.Column("spark_grouping_id"))]
        partial = PL.AggExec(PL.HashAgg, gs, aggs(E.PARTIAL, specs, eschema), False, PL.ExpandExec(eschema, projs, leaf))
        final = PL.AggExec(PL.HashAgg, gs, aggs(E.FINAL, specs, eschema), False, partial)
        got = got_groups(PL.collect(final, conf()), 2)
        keys = [(k, 0) for k in tab.keys] + [(None, 1)] * len(tab.keys)
        cols = {c: v + v for c, v in tab.cols.items()}
        assert_groups(got, X.expected_groups(keys, cols, specs, tab.types), specs, tab.kinds)
        return
    else:
        got, _ = run_one_op(leaf, [], specs, conf())
        got = got_groups(got, 0)
        assert len(got) == 1
        assert_groups(got, expected(tab, specs, grouped=False), specs)
        return
    assert_groups(got_groups(got, 1), expected(tab, specs), specs, tab.kinds)


GROWTH_SHAPES = ["f64 sum avg count", "f64 min max", "dec38_0 sum count", "int sum count"]


@pytest.mark.parametrize("shape", GROWTH_SHAPES)
def test_numeric_edges_through_table_growth(shape):
    """the edge groups among 560 000 single-row groups with sparse keys and NULL arguments: the hashed table grows and the
    deferred rows are replayed; the filler groups are checked in bulk"""
    sh = SHAPES[shape]
    tab = family(sh.family)
    rng = np.random.default_rng(7)
    nfill = 560_000
    fill = np.unique(rng.integers(1 << 40, 1 << 62, nfill, dtype=np.int64))
    fill = fill[rng.permutation(len(fill))]
    rb0 = tab.batches[0]
    filler = pa.RecordBatch.from_arrays([pa.array(fill)] + [pa.nulls(len(fill), rb0.schema.field(i).type) for i in range(1, rb0.num_columns)], schema=rb0.schema)
    half = len(fill) // 2
    batches = [filler.slice(0, half)] + tab.batches + [filler.slice(half)]
    leaf = PL.MemoryExec.from_arrow(batches, tab.schema)
    g = [E.GroupingExpr("k", E.Column("k"))]
    partial = PL.AggExec(PL.HashAgg, g, aggs(E.PARTIAL, sh.specs, leaf.schema()), False, leaf)
    final = PL.AggExec(PL.HashAgg, g, aggs(E.FINAL, sh.specs, leaf.schema()), False, partial)
    out = pa.Table.from_batches(PL.collect(final, conf(agg_initial_groups=1024, max_launch_rows=1 << 16)))
    assert final.last_metrics["table_grow_count"] >= 1
    is_fill = pa.compute.is_in(out.column("k"), value_set=pa.array(fill)).to_numpy(zero_copy_only=False)
    assert int(is_fill.sum()) == len(fill)
    fo = out.filter(pa.array(is_fill))
    for nm, fn, _, _ in sh.specs:
        col = fo.column(nm)
        if fn == E.AGG_COUNT:
            assert col.null_count == 0 and pa.compute.max(col).as_py() == 0
        else:
            assert col.null_count == len(fill), f"{nm}: a filler group with only NULL arguments must be NULL"
    edge = out.filter(pa.array(~is_fill)).to_batches()
    assert_groups(got_groups(edge, 1), expected(tab, sh.specs), sh.specs, tab.kinds)


# ---- Partial state, byte for byte -------------------------------------------------------------------------------------
def _partial_state(tab, specs, cf):
    leaf = PL.MemoryExec.from_arrow(tab.batches, tab.schema)
    g = [E.GroupingExpr("k", E.Column("k"))]
    pa_aggs = aggs(E.PARTIAL, specs, leaf.schema())
    plan = PL.AggExec(PL.HashAgg, g, pa_aggs, False, leaf)
    out = PL.collect(plan, cf)
    oaggs = [O.Agg(a.agg, leaf.schema()) for a in pa_aggs]
    states = {}
    for rb in out:
        keys, bufs = rb.column(0).to_pylist(), rb.column(rb.num_columns - 1).to_pylist()
        for k, buf in zip(keys, bufs):
            accs, pos = [a.create_acc() for a in oaggs], 0
            for a, acc in zip(oaggs, accs):
                pos = a.unfreeze_push(acc, buf, pos)
            assert pos == len(buf)
            states[(k,)] = accs
    return plan, states


def _prim(acc):
    return acc.values[0] if acc.valids[0] else None


@pytest.mark.parametrize("cf", ["default", "generic"])
def test_partial_state_of_negative_zero_sums(cf):
    """the frozen f64 SUM / AVG state of order-independent groups (-0.0 groups among them) is the exact sum, bit for bit"""
    full = family("f64")
    keep = {k for k, kind in full.kinds.items() if kind in ("neg_zero", "neg_zero_nulls", "mixed_zeros", "dyadic", "dyadic_small_row", "subnormal", "all_null")}
    rows = [r for r, k in enumerate(full.keys) if k in keep]
    cols = {"x": [full.cols["x"][r] for r in rows]}
    keys = [full.keys[r] for r in rows]
    rb = pa.RecordBatch.from_arrays([pa.array(keys, pa.int64()), pa.array(cols["x"], pa.float64())], names=["k", "x"])
    n1 = sum(r < full.batches[0].num_rows for r in rows)             # the first batch keeps only dense keys
    tab = X.Table([rb.slice(0, n1), rb.slice(n1)], keys, cols, {"x": F64}, full.kinds)
    specs = [("s", E.AGG_SUM, "x", F64), ("a", E.AGG_AVG, "x", F64)]
    plan, states = _partial_state(tab, specs, conf() if cf == "default" else conf(force_generic_kernels=1))
    if cf == "default":
        assert plan.last_metrics["fast_path_launches"] > 0
    exp = {}
    for k, x in zip(keys, cols["x"]):
        exp.setdefault((k,), []).append(x)
    assert states.keys() == exp.keys()
    bad = []
    for k, xs in exp.items():
        s = X.f64_sum([x for x in xs if x is not None])
        assert s is None or isinstance(s, float)
        n = sum(x is not None for x in xs)
        sacc, (asum, acnt) = states[k]
        for nm, got_v, got_n in (("sum", _prim(sacc), None), ("avg", _prim(asum), acnt.values[0])):
            if not X.matches(s, got_v) or (got_n is not None and got_n != n):
                bad.append((k, full.kinds[k[0]], nm, s, got_v, got_n, n))
    assert not bad, f"{len(bad)} states differ, e.g. {bad[:4]}"


@pytest.mark.parametrize("cf", ["default", "generic"])
def test_partial_state_of_wrapping_decimal_sums(cf):
    """the frozen decimal128 SUM state is the i128-wrapped exact sum of each group"""
    tab = family("dec")
    specs = [("s", E.AGG_SUM, "d0", X.D38_0), ("c", E.AGG_COUNT, "d0", I64)]
    plan, states = _partial_state(tab, specs, conf() if cf == "default" else conf(force_generic_kernels=1))
    if cf == "default":
        assert plan.last_metrics["fast_path_launches"] > 0
    exp = expected(tab, specs)
    assert states.keys() == exp.keys()
    bad = [(k, e, _prim(states[k][0]), states[k][1].values[0]) for k, e in exp.items() if (_prim(states[k][0]), states[k][1].values[0]) != tuple(e)]
    assert not bad, f"{len(bad)} states differ, e.g. {bad[:4]}"
