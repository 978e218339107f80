"""WindowExecNode decode, explain and validation through b200q_plan_explain (no GPU): the decoded node, the rewrites create_agg applies
to window aggregates, and every refusal with its status and reason."""
import pytest

from blaze_b200 import exprs as E, native, plans as PL, proto as P, types as T
from blaze_b200.types import Field, Schema

S = Schema([Field("p", T.int64, True), Field("o", T.int32, False), Field("v", T.int32, True), Field("s", T.utf8, True),
            Field("f", T.float64, True), Field("b", T.bool_, True)])
PART, ORDER = [E.Column("p")], [(E.Column("o"), True, False)]


def explain(exprs, part=PART, order=ORDER, limit=None, owc=True):
    return native.plan_explain(P.window_node(PL.MemoryExec(S).node(), exprs, part, [(e, not d, nf) for e, d, nf in order], limit, owc).SerializeToString())


def refused(code, *a, **k):
    with pytest.raises(native.NativeError) as ei:
        explain(*a, **k)
    assert ei.value.code == code
    return ei.value.msg


def test_explain_prints_the_node():
    txt = explain([E.WindowExpr.rank_like("rk", E.RANK), E.WindowExpr.agg("s", E.AGG_SUM, [E.Column("v")], T.int64),
                   E.WindowExpr.agg("c", E.AGG_COUNT, [E.Column("o"), E.Column("v")], T.int64, False)])
    assert txt.splitlines()[0] == ("WindowExec: [rank() AS rk:int32, SUM(TryCast(v@2 AS int64)) AS s:int64, COUNT(v@2) AS c:int64] "
                                   "partition_by=[p@0] order_by=[o@1 DESC NULLS LAST] output_window_cols=true")
    assert "group_limit=5 output_window_cols=false" in explain([E.WindowExpr.rank_like("rn", E.ROW_NUMBER)], limit=5, owc=False)


def test_schema_is_input_plus_window_columns():
    w = PL.WindowExec(PL.MemoryExec(S), [E.WindowExpr.rank_like("rn", E.ROW_NUMBER)], [], [])
    assert [f.name for f in w.schema()] == [f.name for f in S] + ["rn"]
    assert [f.name for f in PL.WindowExec(PL.MemoryExec(S), [E.WindowExpr.rank_like("rn", E.ROW_NUMBER)], [], [], 3, False).schema()] == [f.name for f in S]


def test_refusals():
    U, I = native.ERR_UNSUPPORTED, native.ERR_INVALID_PLAN
    rn = E.WindowExpr.rank_like("rn", E.ROW_NUMBER)
    assert "FIRST" in refused(U, [E.WindowExpr(Field("x", T.int32, True), E.WINDOW_AGG, agg_func=7, children=[E.Column("v")])])
    assert "COLLECT_LIST" in refused(U, [E.WindowExpr(Field("x", T.int32, True), E.WINDOW_AGG, agg_func=5, children=[E.Column("v")])])
    assert "partition key" in refused(U, [rn], part=[E.Column("s")])
    assert "order key" in refused(U, [rn], order=[(E.Column("s"), False, True)])
    assert "MAX over bool" in refused(U, [E.WindowExpr.agg("m", E.AGG_MAX, [E.Column("b")], T.bool_)])
    assert "MIN over utf8" in refused(U, [E.WindowExpr.agg("m", E.AGG_MIN, [E.Column("s")], T.utf8)])
    assert "its field is int64" in refused(U, [E.WindowExpr(Field("rn", T.int64, False), E.WINDOW_FUNC, window_func=E.ROW_NUMBER, return_type=T.int32)])
    assert "more than 8 window expressions" in refused(U, [E.WindowExpr.rank_like(f"r{i}", E.RANK) for i in range(9)])
    assert "exactly one window expression" in refused(I, [rn, rn], limit=3)
    assert "exactly one window expression" in refused(I, [], limit=3)
    assert "aggregate window column" in refused(U, [E.WindowExpr.agg("s", E.AGG_SUM, [E.Column("v")], T.int64)], limit=3)


def test_order_spec_entry_must_be_a_sort_expression():
    n = P.window_node(PL.MemoryExec(S).node(), [E.WindowExpr.rank_like("rn", E.ROW_NUMBER)], PART, [])
    n.window.order_spec.add().CopyFrom(P.expr_msg(E.Column("o")))          # a bare column, not a PhysicalSortExprNode
    with pytest.raises(native.NativeError) as ei:
        native.plan_explain(n.SerializeToString())
    assert ei.value.code == native.ERR_INVALID_PLAN and "PhysicalSortExprNode" in ei.value.msg
