"""The plan shapes an op's pipeline is built from: where a pending FilterExec / ProjectExec chain becomes its own fused stage (below
SortExec, a hash-join probe, a sort-merge join's left side and ShuffleWriterExec), checked against the oracle, and the shapes op
create and finish refuse, checked by status code and message.

A computed window key under a pending filter and the fused Partial + Final BLOOM_FILTER are covered by
test_gpu_window.py::test_filter_project_window_filter_one_op and test_gpu_bloom.py::test_bloom_agg_fused_partial_final_bytes."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from oracle import blaze_oracle as O
from oracle import join_oracle as J
from oracle import shuffle_oracle as S
from helpers import oracle_batches, parquet_scan, split_batches, with_nulls
from window_cases import window_expr

pytestmark = pytest.mark.gpu
NOSTAGE = native.default_conf(staging_rows=0)


def _table(n, seed, sorted_keys=False):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 300, n, dtype=np.int64)
    if sorted_keys:
        k = np.sort(k)
    v = rng.integers(-1000, 1000, n, dtype=np.int64)
    return pa.RecordBatch.from_arrays([pa.array(k), with_nulls(rng, v, 0.1)], names=["k", "v"])


PRED = [E.BinaryExpr(E.Column("v"), "Gt", E.Literal(-500, T.int64))]
PROJ = [(E.Column("k"), "k"), (E.BinaryExpr(E.Column("v"), "Multiply", E.Literal(3, T.int64)), "v3")]


def _filter_project(batches):
    """FilterExec -> ProjectExec over the batches: the plan, and the oracle's rows"""
    leaf = PL.MemoryExec.from_arrow(batches, batches[0].schema)
    plan = PL.ProjectExec(PROJ, PL.FilterExec(PRED, leaf))
    ins = leaf.schema()
    exp = O.ProjectExec(PROJ, ins).execute(O.FilterExec(PRED, ins).execute(oracle_batches(batches)))
    return plan, exp


def _error(fn):
    with pytest.raises(native.NativeError) as e:
        fn()
    return e.value.code, e.value.msg


def _create_error(plan):
    def create():
        native.NativeOp(plan.plan_bytes(), NOSTAGE).close()
    return _error(create)


# ---- a pending Filter -> Project chain below the operators that take it as their own stage ----------------------------------------
def test_filter_project_below_sort():
    batches = split_batches(_table(3_000, 1), 700)
    fp, exp = _filter_project(batches)
    plan = PL.SortExec(fp, [(E.Column("k"), False, True), (E.Column("v3"), True, True)])
    got = [tuple(r.values()) for b in PL.collect(plan, NOSTAGE) for r in b.to_pylist()]
    want = [tuple(r.values()) for b in exp for r in O.batch_to_arrow(b).to_pylist()]
    want.sort(key=lambda r: (r[0], r[1] is not None, -r[1] if r[1] is not None else 0))      # k ascending, then v3 descending, NULLs first
    assert got == want


def test_filter_project_below_a_hash_join_probe():
    lb, rb = split_batches(_table(3_000, 2), 700), [_table(500, 3).rename_columns(["kr", "vr"])]
    fp, exp_left = _filter_project(lb)
    build = PL.MemoryExec.from_arrow(rb, rb[0].schema)
    schema = PL.build_join_schema(fp.schema(), build.schema(), PL.JOIN_INNER)
    plan = PL.BroadcastJoinExec(schema, fp, build, [(E.Column("k"), E.Column("kr"))], PL.JOIN_INNER, PL.RIGHT_SIDE)
    got = PL.collect(plan, NOSTAGE)
    exp = J.HashJoin(fp.schema(), build.schema(), [(0, 0)], J.INNER, "right").execute(exp_left, oracle_batches(rb))
    assert O.rows_multiset([O.batch_from_arrow(b) for b in got]) == O.rows_multiset(exp)


def test_filter_project_below_a_sort_merge_join_left_side():
    # keys sorted on both sides; the filter and the projection keep the left side sorted, so no SortExec sits between them and the join
    lb, rb = split_batches(_table(3_000, 4, sorted_keys=True), 700), [_table(500, 5, sorted_keys=True).rename_columns(["kr", "vr"])]
    fp, exp_left = _filter_project(lb)
    right = PL.MemoryExec.from_arrow(rb, rb[0].schema)
    schema = PL.build_join_schema(fp.schema(), right.schema(), PL.JOIN_INNER)
    plan = PL.SortMergeJoinExec(schema, fp, right, [(E.Column("k"), E.Column("kr"))], [(True, True)], PL.JOIN_INNER)
    got = PL.collect(plan, NOSTAGE)
    exp = J.HashJoin(fp.schema(), right.schema(), [(0, 0)], J.INNER, "right").execute(exp_left, oracle_batches(rb))
    assert O.rows_multiset([O.batch_from_arrow(b) for b in got]) == O.rows_multiset(exp)


def test_filter_project_below_a_shuffle_writer(tmp_path):
    batches = split_batches(_table(3_000, 6), 700)
    fp, exp = _filter_project(batches)
    plan = PL.ShuffleWriterExec(fp, ("single",), str(tmp_path / "s.data"), str(tmp_path / "s.index"))
    PL.collect(plan, NOSTAGE)
    parts = S.read_shuffle_file(open(plan.output_data_file, "rb").read(), open(plan.output_index_file, "rb").read(), fp.schema())
    assert len(parts) == 1 and O.rows_multiset(parts[0]) == O.rows_multiset(exp)


# ---- shapes the pipeline refuses ---------------------------------------------------------------------------------------------
def test_parquet_scan_of_a_utf8_column_is_unsupported(tmp_path):
    t = pa.table({"k": pa.array([1, 2, 3], pa.int64()), "s": pa.array(["a", "b", None], pa.string())})
    path = str(tmp_path / "s.parquet")
    pq.write_table(t, path)
    code, msg = _create_error(parquet_scan(path, t.schema))
    assert code == native.ERR_UNSUPPORTED and "BYTE_ARRAY decode is not on the GPU path" in msg


def test_projection_below_a_merge_mode_aggregate_is_unsupported():
    rb = _table(100, 7)
    ins = T.from_arrow_schema(rb.schema)
    g = [E.GroupingExpr("k", E.Column("k"))]
    partial = PL.AggExec(PL.HashAgg, g, [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], ins, T.int64))], False, PL.MemoryExec(ins))
    states = PL.MemoryExec(partial.schema())
    proj = PL.ProjectExec([(E.BinaryExpr(E.Column("k"), "Plus", E.Literal(1, T.int64)), "k"), (E.Column(E.AGG_BUF_COLUMN_NAME), E.AGG_BUF_COLUMN_NAME)], states)
    final = PL.AggExec(PL.HashAgg, g, [E.AggExpr("s", E.FINAL, PL.create_agg(E.AGG_SUM, [E.placeholder(T.int64)], ins, T.int64))], False, proj)
    code, msg = _create_error(final)
    assert code == native.ERR_UNSUPPORTED and "Projection fused below a merge-mode aggregate" in msg


def _bloom(mode, child, schema):
    return [E.AggExpr("bf", mode, PL.create_agg(E.AGG_BLOOM_FILTER, [child, E.Literal(5_000, T.int64), E.Literal(1 << 16, T.int64)], schema, T.binary))]


@pytest.mark.parametrize("below", ["filter", "projection"])
def test_filter_or_projection_below_a_merge_mode_bloom_filter_is_unsupported(below):
    ks = T.Schema([T.Field("k", T.int64, True)])
    partial = PL.AggExec(PL.HashAgg, [], _bloom(E.PARTIAL, E.XxHash64(E.Column("k")), ks), False, PL.MemoryExec(ks))
    states = PL.MemoryExec(partial.schema())
    buf = E.Column(E.AGG_BUF_COLUMN_NAME)
    if below == "filter":
        src = PL.FilterExec([E.IsNotNull(buf)], states)
    else:                                                           # a projection that is not the identity: the column twice
        src = PL.ProjectExec([(buf, "x"), (buf, E.AGG_BUF_COLUMN_NAME)], states)
    final = PL.AggExec(PL.HashAgg, [], _bloom(E.FINAL, E.placeholder(T.binary), ks), False, src)
    code, msg = _create_error(final)
    assert code == native.ERR_UNSUPPORTED and "Filter / Projection fused below a merge-mode BLOOM_FILTER aggregate" in msg


def test_join_build_below_another_operator_is_unsupported():
    leaf = PL.MemoryExec(T.from_arrow_schema(_table(10, 8).schema))
    build = PL.BroadcastJoinBuildHashMapExec(leaf, [E.Column("k")])
    code, msg = _create_error(PL.ProjectExec([(E.Column("k"), "k")], build))
    assert code == native.ERR_UNSUPPORTED and "BroadcastJoinBuildHashMapExec below another operator" in msg


def test_shuffle_writer_below_another_operator_is_unsupported(tmp_path):
    leaf = PL.MemoryExec(T.from_arrow_schema(_table(10, 9).schema))
    writer = PL.ShuffleWriterExec(leaf, ("single",), str(tmp_path / "s.data"), str(tmp_path / "s.index"))
    code, msg = _create_error(PL.ProjectExec([(E.Column("k"), "k")], writer))
    assert code == native.ERR_UNSUPPORTED and "ShuffleWriterExec below another operator" in msg


def test_window_over_a_group_limit_that_outputs_its_window_column_is_unsupported():
    rb = _table(100, 10, sorted_keys=True)
    schema = T.from_arrow_schema(rb.schema)
    part, order = [E.Column("k")], [(E.Column("v"), False, True)]
    child = PL.WindowExec(PL.MemoryExec(schema), [window_expr("w", "rank", None, schema)], part, order, 3, True)
    parent = PL.WindowExec(child, [window_expr("rk", "row_number", None, schema)], part, order)
    code, msg = _create_error(parent)
    assert code == native.ERR_UNSUPPORTED and "outputs its window column" in msg


def test_a_parquet_scan_op_takes_no_pushed_batches(tmp_path):
    rb = _table(100, 11)
    path = str(tmp_path / "k.parquet")
    pq.write_table(pa.Table.from_batches([rb]), path)
    with native.NativeOp(parquet_scan(path, rb.schema).plan_bytes(), NOSTAGE) as op:
        op.push(rb)
        code, msg = _error(op.finish)
    assert code == native.ERR_STATE and "takes no pushed batches" in msg
