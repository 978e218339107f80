"""ExpandExecNode decoding and validation in the native library (no GPU needed: plans are decoded by b200q_plan_explain)."""
import pytest

from blaze_b200 import exprs as E, native, plans as PL, proto as P, types as T
from blaze_b200.types import Field, Schema

from expand_cases import expand_for_sets, grouping_sets

IN = Schema([Field("k1", T.int64, False), Field("k2", T.int32, True), Field("v", T.int64, True), Field("s", T.utf8, True)])


def leaf():
    return PL.MemoryExec(IN)


def test_decode_and_explain():
    schema, projs = expand_for_sets(IN, ["k1", "k2"], ["v", "s"], grouping_sets("rollup", 2))
    ex = PL.ExpandExec(schema, projs, leaf())
    text = ex.explain()
    first = text.splitlines()[0]
    assert first.startswith("ExpandExec projections=[[k1@0 AS k1, k2@1 AS k2, v@2 AS v, s@3 AS s, 0:int64 AS spark_grouping_id], ")
    assert "[NULL:int64 AS k1, NULL:int32 AS k2, v@2 AS v, s@3 AS s, 3:int64 AS spark_grouping_id]" in first
    assert "schema=[k1:int64?, k2:int32?, v:int64?, s:utf8?, spark_grouping_id:int64]" in first
    assert text.splitlines()[1].strip().startswith("FFIReader")


def test_expand_below_partial_aggregate_decodes():
    schema, projs = expand_for_sets(IN, ["k1", "k2"], ["v"], grouping_sets("cube", 2))
    ex = PL.ExpandExec(schema, projs, leaf())
    g = [E.GroupingExpr(n, E.Column(n)) for n in ("k1", "k2", "spark_grouping_id")]
    a = [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], schema, T.int64))]
    text = PL.AggExec(PL.HashAgg, g, a, False, ex).explain()
    assert text.splitlines()[1].strip().startswith("ExpandExec")


def _raises(code, match, fn):
    with pytest.raises(native.NativeError) as ei:
        fn()
    assert ei.value.code == code and match in ei.value.msg, ei.value.msg


def test_type_mismatch_is_invalid_plan():
    s = Schema([Field("k1", T.int32, False)])
    _raises(native.ERR_INVALID_PLAN, "ExpandExec data type not matches: Some(int64) vs int32",
            lambda: PL.ExpandExec(s, [[E.Column("k1")]], leaf()))


def test_short_projection_is_invalid_plan():
    s = Schema([Field("k1", T.int64, False), Field("v", T.int64, True)])
    _raises(native.ERR_INVALID_PLAN, "ExpandExec data type not matches: None vs int64",
            lambda: PL.ExpandExec(s, [[E.Column("k1"), E.Column("v")], [E.Column("k1")]], leaf()))


def test_missing_input_or_schema_is_invalid_plan():
    n = P.PhysicalPlanNode()
    n.expand.schema.CopyFrom(P.schema_msg(IN))
    _raises(native.ERR_INVALID_PLAN, "Missing required field", lambda: native.plan_explain(n.SerializeToString()))


def test_extra_expressions_are_ignored():
    s = Schema([Field("k1", T.int64, False)])
    ex = PL.ExpandExec(s, [[E.Column("k1"), E.Column("v"), E.Literal(1, T.int32)]], leaf())
    assert ex.explain().splitlines()[0] == "ExpandExec projections=[[k1@0 AS k1]] schema=[k1:int64]"


def test_zero_projections_accepted():
    s = Schema([Field("k1", T.int64, False)])
    assert PL.ExpandExec(s, [], leaf()).explain().splitlines()[0] == "ExpandExec projections=[] schema=[k1:int64]"


def test_tag_20_is_expand_in_the_proto_mirror():
    assert P.PhysicalPlanNode.DESCRIPTOR.fields_by_name["expand"].number == 20
    assert [f.name for f in P.PhysicalPlanNode.ExpandExecNode.DESCRIPTOR.fields] == ["input", "schema", "projections"]
    assert [f.name for f in P.PhysicalPlanNode.ExpandProjection.DESCRIPTOR.fields] == ["expr"]
