"""ExpandExec on the GPU against the oracle: the reference's KATs, the standalone path (every input batch yields its projections in
order), and ROLLUP / CUBE / GROUPING SETS / multi-DISTINCT Expands fused into AggExec(Partial), through Final in two ops, fused in one
op, and on the map side of a shuffle.  Run again with B200Q_NO_AGG_FUSION=1 to keep Partial and Final in separate stages."""
import decimal
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from blaze_b200.types import Field, Schema
from oracle import blaze_oracle as O
from oracle import expand_oracle as X
from oracle import shuffle_oracle as S
from helpers import *
from expand_cases import KATS, expand_for_sets, grouping_sets, kat_input, kat_projections, kat_text

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNSTAGED = dict(staging_rows=0)          # every pushed batch reaches the stages as it is: the per-batch projection order is observable


def conf(**kw):
    return native.default_conf(**kw)


# ---- the reference's KATs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", KATS, ids=[c["name"] for c in KATS])
def test_kats(case):
    schema, rb = kat_input(case)
    out = PL.collect(PL.ExpandExec(schema, kat_projections(case), PL.MemoryExec.from_arrow([rb])))
    assert [b.num_rows for b in out] == [4] * len(case["expected"])          # one batch per projection, in order
    for b, exp in zip(out, case["expected"]):
        assert b.column(0).null_count == 0
        assert kat_text(case, b.column(0).to_pylist()) == exp


# ---- the standalone path -------------------------------------------------------------------------------------------------------
def _int_input(n=20_000, seed=3):
    rng = np.random.default_rng(seed)
    return pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 30, n, dtype=np.int64)), with_nulls(rng, rng.integers(-5, 5, n).astype(np.int32), 0.2),
                                       with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.1), pa.array(rng.integers(0, 100, n, dtype=np.int64))],
                                      names=["k1", "k2", "v", "f"])


def _standalone_projections(ins):
    schema, projs = expand_for_sets(ins, ["k1", "k2"], ["v"], grouping_sets("rollup", 2))
    projs[0][2] = E.BinaryExpr(E.Column("v"), "Multiply", E.Literal(3, T.int64))          # a computed column in one set
    return schema, projs


def test_expand_at_the_top_keeps_projection_order():
    rb = _int_input()
    batches = split_batches(rb, 3_000)
    ins = T.from_arrow_schema(rb.schema)
    schema, projs = _standalone_projections(ins)
    got = PL.collect(PL.ExpandExec(schema, projs, PL.MemoryExec.from_arrow(batches, rb.schema)), conf(**UNSTAGED))
    exp = X.ExpandExec(schema, projs, ins).execute(oracle_batches(batches))
    assert [b.num_rows for b in got] == [b.num_rows for b in exp]
    assert_same_rows_ordered(got, exp, schema)
    # staged host batches: same rows
    assert_multiset_equal(PL.collect(PL.ExpandExec(schema, projs, PL.MemoryExec.from_arrow(batches, rb.schema))), exp)


def test_expand_over_filter_and_project_below():
    rb = _int_input(seed=4)
    batches = split_batches(rb, 4_000)
    ins = T.from_arrow_schema(rb.schema)
    preds = [E.BinaryExpr(E.Column("f"), "Lt", E.Literal(60, T.int64))]
    below = [(E.Column("k1"), "k1"), (E.Column("k2"), "k2"), (E.BinaryExpr(E.Column("v"), "Minus", E.Column("f")), "v")]
    proj = PL.ProjectExec(below, PL.FilterExec(preds, PL.MemoryExec.from_arrow(batches, rb.schema)))
    schema, projs = _standalone_projections(proj.schema())
    got = PL.collect(PL.ExpandExec(schema, projs, proj), conf(**UNSTAGED))
    op = O.ProjectExec(below, ins, preds)
    exp = X.ExpandExec(schema, projs, op.schema).execute(op.execute(oracle_batches(batches)))
    assert_same_rows_ordered(got, exp, schema)


def test_filter_above_expand():
    rb = _int_input(seed=5)
    batches = split_batches(rb, 5_000)
    ins = T.from_arrow_schema(rb.schema)
    schema, projs = _standalone_projections(ins)
    pred = [E.SCOr(E.BinaryExpr(E.Column("spark_grouping_id"), "Eq", E.Literal(3, T.int64)), E.BinaryExpr(E.Column("v"), "Gt", E.Literal(0, T.int64)))]
    got = PL.collect(PL.FilterExec(pred, PL.ExpandExec(schema, projs, PL.MemoryExec.from_arrow(batches, rb.schema))), conf(**UNSTAGED))
    exp = O.FilterExec(pred, schema).execute(X.ExpandExec(schema, projs, ins).execute(oracle_batches(batches)))
    assert_same_rows_ordered(got, exp, schema)


def test_expand_into_shuffle_writer(tmp_path):
    rb = _int_input(seed=6)
    batches = split_batches(rb, 5_000)
    ins = T.from_arrow_schema(rb.schema)
    schema, projs = _standalone_projections(ins)
    w = PL.ShuffleWriterExec(PL.ExpandExec(schema, projs, PL.MemoryExec.from_arrow(batches, rb.schema)), ("hash", [E.Column("k1")], 7),
                             str(tmp_path / "e.data"), str(tmp_path / "e.index"))
    PL.collect(w)
    parts = S.read_shuffle_file(open(w.output_data_file, "rb").read(), open(w.output_index_file, "rb").read(), schema)
    exp = X.ExpandExec(schema, projs, ins).execute(oracle_batches(batches))
    assert O.rows_multiset([b for p in parts for b in p]) == O.rows_multiset(exp)
    for q, p in enumerate(parts):                                          # each partition holds exactly the rows murmur3 sends there
        for b in p:
            assert (O.partition_ids(O.create_murmur3_hashes([b.cols[0]], b.num_rows), 7) == q).all()


def test_expand_carries_utf8_columns():
    rng = np.random.default_rng(8)
    n = 5_000
    words = ["", "a", "héllo", "x" * 70, "rollup"]
    s = [None if rng.random() < 0.1 else words[i] for i in rng.integers(0, len(words), n)]
    k = rng.integers(0, 9, n, dtype=np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(k), pa.array(s, pa.string())], names=["k", "s"])
    batches = split_batches(rb, 1_500)
    ins = T.from_arrow_schema(rb.schema)
    schema, projs = expand_for_sets(ins, ["k"], ["s"], grouping_sets("rollup", 1))
    got = PL.collect(PL.ExpandExec(schema, projs, PL.MemoryExec.from_arrow(batches, rb.schema)), conf(**UNSTAGED))
    exp = []
    for b in batches:
        kk, ss = b.column(0).to_pylist(), b.column(1).to_pylist()
        exp.append(list(zip(kk, ss, [0] * len(kk))))
        exp.append(list(zip([None] * len(kk), ss, [1] * len(kk))))
    assert [list(zip(*[c.to_pylist() for c in g.columns])) for g in got] == exp


# ---- Expand fused into AggExec(Partial) ----------------------------------------------------------------------------------------
SPECS = [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, "v", T.int64), ("a", E.AGG_AVG, "x", T.float64), ("mn", E.AGG_MIN, "v", T.int64),
         ("mx", E.AGG_MAX, "x", T.float64), ("sd", E.AGG_SUM, "d", T.decimal128(27, 2)), ("ad", E.AGG_AVG, "d", T.decimal128(21, 6)),
         ("md", E.AGG_MAX, "d", T.decimal128(17, 2))]


def _key_array(rng, kind, n, nullable):
    if kind == "int64":
        a, t = rng.integers(0, 40, n, dtype=np.int64), None
    elif kind == "int32":
        a, t = rng.integers(-6, 6, n).astype(np.int32), None
    elif kind == "date32":
        a, t = rng.integers(18_000, 18_012, n).astype(np.int32), pa.date32()
    else:
        a, t = [decimal.Decimal(int(x)).scaleb(-2) for x in rng.integers(-400, 400, n)], pa.decimal128(9, 2)
    if nullable:
        return pa.array(a, mask=rng.random(n) < 0.1, type=t)
    return pa.array(a, type=t)


def _agg_input(key_kinds, nullable, n=24_000, seed=11):
    rng = np.random.default_rng(seed)
    raw = rng.integers(-10**12, 10**12, n)
    cols = [_key_array(rng, kk, n, nullable) for kk in key_kinds]
    cols += [with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.1), with_nulls(rng, rng.normal(0, 1e6, n), 0.1),
             pa.array([decimal.Decimal(int(r)).scaleb(-2) for r in raw], pa.decimal128(17, 2)), pa.array(rng.integers(0, 100, n, dtype=np.int64))]
    names = [f"k{i + 1}" for i in range(len(key_kinds))] + ["v", "x", "d", "f"]
    return pa.RecordBatch.from_arrays(cols, names=names)


def _aggs(mode, specs, ins):
    if mode == E.PARTIAL:
        return [E.AggExpr(nm, mode, PL.create_agg(fn, [E.Column(c)], ins, rt)) for nm, fn, c, rt in specs]
    by_name = {f.name: f.dtype for f in ins}
    return [E.AggExpr(nm, mode, PL.create_agg(fn, [E.placeholder(by_name[c])], ins, rt)) for nm, fn, c, rt in specs]


class Fused:
    """Filter -> Project -> Expand(sets) -> AggExec(Partial) [-> AggExec(Final)] over `rb`, and the oracle's answer"""

    def __init__(self, rb, nkeys, sets, gid_type=T.int64, specs=SPECS, batch_rows=5_000):
        self.rb, self.batches = rb, split_batches(rb, batch_rows)
        self.ins = T.from_arrow_schema(rb.schema)
        keys = [f"k{i + 1}" for i in range(nkeys)]
        self.preds = [E.BinaryExpr(E.Column("f"), "Lt", E.Literal(70, T.int64))]
        self.below = [(E.Column(k), k) for k in keys] + [(E.BinaryExpr(E.Column("v"), "Plus", E.Literal(1, T.int64)), "v"), (E.Column("x"), "x"), (E.Column("d"), "d")]
        self.proj_schema = O.ProjectExec(self.below, self.ins).schema
        self.eschema, self.projs = expand_for_sets(self.proj_schema, keys, ["v", "x", "d"], sets, gid_type)
        self.g = [E.GroupingExpr(n, E.Column(n)) for n in keys + ["spark_grouping_id"]]
        self.specs, self.nk = specs, nkeys + 1

    def expand(self, leaf):
        return PL.ExpandExec(self.eschema, self.projs, PL.ProjectExec(self.below, PL.FilterExec(self.preds, leaf)))

    def partial(self, leaf, columnar=False):
        return PL.AggExec(PL.HashAgg, self.g, _aggs(E.PARTIAL, self.specs, self.eschema), False, self.expand(leaf), columnar_state=columnar)

    def final_over(self, child_plan, pschema):
        return PL.AggExec(PL.HashAgg, self.g, _aggs(E.FINAL, self.specs, self.eschema), False, child_plan)

    def leaf(self, batches=None):
        return PL.MemoryExec.from_arrow(batches if batches is not None else self.batches, self.rb.schema)

    def oracle(self, batches=None):
        op0 = O.ProjectExec(self.below, self.ins, self.preds)
        ex = X.ExpandExec(self.eschema, self.projs, op0.schema)
        op = O.AggExec(E.HASH_AGG, self.g, _aggs(E.PARTIAL, self.specs, self.eschema), False, self.eschema)
        of = O.AggExec(E.HASH_AGG, self.g, _aggs(E.FINAL, self.specs, self.eschema), False, op.schema)
        return of.execute(op.execute(ex.execute(op0.execute(oracle_batches(batches if batches is not None else self.batches)))))

    def float_cols(self):
        return tuple(self.nk + i for i, s in enumerate(self.specs) if s[0] in ("a", "mx"))

    def two_ops(self, cf=None, columnar=False):
        partial = self.partial(self.leaf(), columnar)
        parts = PL.collect(partial, cf)
        return PL.collect(self.final_over(PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(partial.schema())), partial.schema()), cf)

    def one_op(self, cf=None):
        partial = self.partial(self.leaf())
        return PL.collect(self.final_over(partial, partial.schema()), cf)


SHAPES = {
    "rollup-i64": (["int64"], False, grouping_sets("rollup", 1), T.int64),
    "rollup-i64-i32": (["int64", "int32"], False, grouping_sets("rollup", 2), T.int64),
    "rollup-date-dec-null": (["date32", "decimal"], True, grouping_sets("rollup", 2), T.int32),
    "cube-i32-date-dec": (["int32", "date32", "decimal"], True, grouping_sets("cube", 3), T.int64),
    "sets-i64-i32-date": (["int64", "int32", "date32"], True, [(0, 1), (2,), (0,), ()], T.int32),
}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("form", ["two_ops", "one_op", "columnar"])
def test_rollup_cube_grouping_sets(shape, form):
    kinds, nullable, sets, gid = SHAPES[shape]
    fx = Fused(_agg_input(kinds, nullable, seed=len(shape)), len(kinds), sets, gid)
    if form == "two_ops":
        got = fx.two_ops()
    elif form == "one_op":
        got = fx.one_op()
    else:
        got = fx.two_ops(conf(partial_state_columnar=1), columnar=True)
    assert_multiset_equal(got, fx.oracle(), float_cols=fx.float_cols())


def test_fused_partial_keeps_the_grouping_set_kernel():
    """the Expand is fused: no ExpandExec stage materialises the sets (one VM launch per chunk covers every set)"""
    fx = Fused(_agg_input(["int64", "int32"], False), 2, grouping_sets("rollup", 2))
    partial = fx.partial(fx.leaf())
    PL.collect(partial)
    m = partial.last_metrics
    assert m["fast_path_launches"] == 0
    assert m["hot_kernel_rows"] == fx.rb.num_rows                 # stage 0 is the aggregate: it read each input row once, not rows x sets


@pytest.mark.skipif(os.environ.get("B200Q_NO_AGG_FUSION") is not None, reason="already without Partial/Final fusion")
def test_shapes_again_without_partial_final_fusion():
    env = dict(os.environ, B200Q_NO_AGG_FUSION="1")
    r = subprocess.run([sys.executable, "-m", "pytest", __file__, "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "rollup_cube_grouping_sets and one_op"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ---- the multi-DISTINCT rewrite (RewriteDistinctAggregates): the first level groups by (k, a, b, gid) ---------------------------
def _distinct_input(n=20_000, seed=21):
    rng = np.random.default_rng(seed)
    return pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 50, n, dtype=np.int64)), with_nulls(rng, rng.integers(0, 30, n).astype(np.int32), 0.1),
                                       with_nulls(rng, rng.integers(-20, 20, n, dtype=np.int64), 0.1), with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.1)],
                                      names=["k", "a", "b", "v"])


def _distinct_plan(rb, with_regular):
    ins = T.from_arrow_schema(rb.schema)
    fields = [Field("k", T.int64, False), Field("a", T.int32, True), Field("b", T.int64, True), Field("gid", T.int64, False)]
    n32, n64 = E.Literal(None, T.int32), E.Literal(None, T.int64)
    projs = [[E.Column("k"), E.Column("a"), n64, E.Literal(1, T.int64)], [E.Column("k"), n32, E.Column("b"), E.Literal(2, T.int64)]]
    if with_regular:
        fields.append(Field("v", T.int64, True))
        projs = [p + [n64] for p in projs] + [[E.Column("k"), n32, n64, E.Literal(0, T.int64), E.Column("v")]]
    schema = Schema(fields)
    g = [E.GroupingExpr(n, E.Column(n)) for n in ("k", "a", "b", "gid")]
    specs = [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, "v", T.int64)] if with_regular else []
    return ins, schema, projs, g, specs


@pytest.mark.parametrize("with_regular", [False, True], ids=["distinct_only", "with_regular_agg"])
@pytest.mark.parametrize("fused_final", [False, True], ids=["two_ops", "one_op"])
def test_multi_distinct_first_level(with_regular, fused_final):
    rb = _distinct_input()
    batches = split_batches(rb, 6_000)
    ins, schema, projs, g, specs = _distinct_plan(rb, with_regular)
    partial = PL.AggExec(PL.HashAgg, g, _aggs(E.PARTIAL, specs, schema), False, PL.ExpandExec(schema, projs, PL.MemoryExec.from_arrow(batches, rb.schema)))
    if fused_final:
        got = PL.collect(PL.AggExec(PL.HashAgg, g, _aggs(E.FINAL, specs, schema), False, partial))
    else:
        parts = PL.collect(partial)
        got = PL.collect(PL.AggExec(PL.HashAgg, g, _aggs(E.FINAL, specs, schema), False, PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(partial.schema()))))
    op = O.AggExec(E.HASH_AGG, g, _aggs(E.PARTIAL, specs, schema), False, schema)
    of = O.AggExec(E.HASH_AGG, g, _aggs(E.FINAL, specs, schema), False, op.schema)
    exp = of.execute(op.execute(X.ExpandExec(schema, projs, ins).execute(oracle_batches(batches))))
    assert_multiset_equal(got, exp)


# ---- the map side: Expand -> AggExec(Partial) -> ShuffleWriterExec, reduced by the GPU AggExec(Final) -----------------------------
def test_map_side_then_final_reduce(tmp_path):
    fx = Fused(_agg_input(["int64", "int32"], True, n=30_000, seed=31), 2, grouping_sets("rollup", 2))
    P = 9
    hash_keys = [E.Column("k1"), E.Column("k2"), E.Column("spark_grouping_id")]
    maps = []
    for m, (lo, hi) in enumerate(((0, 11_000), (11_000, 30_000))):
        partial = fx.partial(fx.leaf(split_batches(fx.rb.slice(lo, hi - lo), 5_000)))
        w = PL.ShuffleWriterExec(partial, ("hash", hash_keys, P), str(tmp_path / f"m{m}.data"), str(tmp_path / f"m{m}.index"))
        PL.collect(w, native.default_conf())                                   # reference format: keys + Binary accumulator rows
        maps.append(S.read_shuffle_file(open(w.output_data_file, "rb").read(), open(w.output_index_file, "rb").read(), partial.schema()))
    pschema = partial.schema()
    got = []
    for q in range(P):
        parts = [O.batch_to_arrow(b) for mp in maps for b in mp[q]]
        if parts:
            got += PL.collect(fx.final_over(PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(pschema)), pschema))
    assert_multiset_equal(got, fx.oracle([fx.rb]), float_cols=fx.float_cols())


# ---- growth with deferred (row, set) pairs ----------------------------------------------------------------------------------------
def test_growth_with_sets_in_different_launches():
    """CUBE over two unique keys: 3 groups per row, far beyond the first table (2^20 slots, load limit 2^19), two growths.
    Small launches put the sets of one row's neighbours in different launches; exact int64 sums catch a set counted twice."""
    rng = np.random.default_rng(41)
    n = 600_000
    rb = pa.RecordBatch.from_arrays([pa.array(rng.permutation(n).astype(np.int64)), pa.array(rng.permutation(n).astype(np.int64)),
                                     pa.array(rng.integers(-2**40, 2**40, n, dtype=np.int64)), pa.array(rng.normal(0, 1, n)),
                                     pa.array([decimal.Decimal(1)] * n, pa.decimal128(17, 2)), pa.array(np.zeros(n, dtype=np.int64))],
                                    names=["k1", "k2", "v", "x", "d", "f"])
    specs = [("s", E.AGG_SUM, "v", T.int64), ("c", E.AGG_COUNT, "v", T.int64)]
    fx = Fused(rb, 2, grouping_sets("cube", 2), specs=specs, batch_rows=200_000)
    cf = conf(agg_initial_groups=1000, max_launch_rows=1 << 16)
    partial = fx.partial(fx.leaf())
    parts = PL.collect(partial, cf)
    assert partial.last_metrics["table_grow_count"] >= 2
    got = PL.collect(fx.final_over(PL.MemoryExec.from_arrow(parts, T.to_arrow_schema(partial.schema())), partial.schema()), cf)
    assert_multiset_equal(got, fx.oracle())


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
def test_operator_outside_the_vm_is_refused():
    rb = _int_input(n=100)
    ins = T.from_arrow_schema(rb.schema)
    leaf = PL.MemoryExec.from_arrow([rb])
    # a Spark extension function the device evaluator does not have, in one set: refused, standalone and below an aggregate alike
    s1 = Schema([Field("k1", T.int64, True), Field("gid", T.int64, False)])
    projs = [[E.Column("k1"), E.Literal(0, T.int64)], [E.ScalarFunction("Spark_NotOnTheDevice", [E.Column("k1")], T.int64), E.Literal(1, T.int64)]]
    g = [E.GroupingExpr("k1", E.Column("k1")), E.GroupingExpr("gid", E.Column("gid"))]
    for build in (lambda: PL.ExpandExec(s1, projs, leaf), lambda: PL.AggExec(PL.HashAgg, g, [], False, PL.ExpandExec(s1, projs, leaf))):
        with pytest.raises(native.NativeError) as ei:
            PL.collect(build())
        assert ei.value.code == native.ERR_UNSUPPORTED and "Spark_NotOnTheDevice" in ei.value.msg
    # a Utf8 value other than a column reference: ProjectExec refuses it, so does the Expand
    s = Schema([Field("k1", T.int64, False), Field("s", T.utf8, True)])
    plan = PL.ExpandExec(s, [[E.Column("k1"), E.Literal(None, T.utf8)], [E.Column("k1"), E.Literal(None, T.utf8)]], leaf)
    with pytest.raises(native.NativeError) as ei:
        PL.collect(plan)
    assert ei.value.code == native.ERR_UNSUPPORTED and "ProjectExec" in ei.value.msg


def test_set_limit():
    rb = _int_input(n=2_000)
    ins = T.from_arrow_schema(rb.schema)
    leaf = lambda: PL.MemoryExec.from_arrow([rb])

    def plan(nsets):
        schema = Schema([Field("k1", T.int64, False), Field("v", T.int64, True), Field("gid", T.int64, False)])
        projs = [[E.Column("k1"), E.Column("v"), E.Literal(i, T.int64)] for i in range(nsets)]
        g = [E.GroupingExpr("k1", E.Column("k1")), E.GroupingExpr("gid", E.Column("gid"))]
        return schema, projs, PL.AggExec(PL.HashAgg, g, _aggs(E.PARTIAL, [("s", E.AGG_SUM, "v", T.int64)], schema), False,
                                         PL.ExpandExec(schema, projs, leaf()))
    with pytest.raises(native.NativeError) as ei:
        PL.collect(plan(65)[2])
    assert ei.value.code == native.ERR_UNSUPPORTED and "64 grouping sets" in ei.value.msg
    # 64 sets fuse; the same 65 projections standalone (no aggregate above) are not limited
    schema, projs, p = plan(64)
    parts = PL.collect(p)
    assert sum(b.num_rows for b in parts) == 64 * len(set(rb.column(0).to_pylist()))
    out = PL.collect(PL.ExpandExec(schema, plan(65)[1], leaf()), conf(**UNSTAGED))
    assert sum(b.num_rows for b in out) == 65 * rb.num_rows


def test_zero_projections_yield_no_rows():
    rb = _int_input(n=1_000)
    s = Schema([Field("k1", T.int64, False)])
    assert PL.collect(PL.ExpandExec(s, [], PL.MemoryExec.from_arrow([rb]))) == []
    g = [E.GroupingExpr("k1", E.Column("k1"))]
    assert PL.collect(PL.AggExec(PL.HashAgg, g, [], False, PL.ExpandExec(s, [], PL.MemoryExec.from_arrow([rb])))) == []
