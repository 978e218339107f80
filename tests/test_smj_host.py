"""SortMergeJoinExec without a GPU: decoding and explaining the SortMergeJoinExecNode (plan node #10), and every validation and
refusal of the node — through the explain entry point and through op create, which decodes the plan before it looks for a device."""
import pytest

from blaze_b200 import exprs as E, native, plans as PL, proto as P, types as T
from blaze_b200.types import Field, Schema

LS = Schema([Field("k", T.int64, True), Field("j", T.int32, True), Field("v", T.float64, True)])
RS = Schema([Field("rk", T.int64, True), Field("rj", T.int32, True), Field("w", T.decimal128(20, 2), True)])
ASC_NF = (True, True)


def _leaf(s, rid):
    return PL.MemoryExec(s, resource_id=rid)


def _node(on, sort_options, jt=PL.JOIN_INNER, ls=LS, rs=RS, schema=None):
    schema = schema if schema is not None else PL.build_join_schema(ls, rs, jt)
    return P.smj_node(schema, _leaf(ls, "l").node(), _leaf(rs, "r").node(), on, sort_options, jt)


def _err(node):
    b = node.SerializeToString()
    with pytest.raises(native.NativeError) as ei:
        native.plan_explain(b)
    with pytest.raises(native.NativeError) as ec:                      # op create decodes first: the same refusal without a GPU
        native.NativeOp(b)
    assert (ec.value.code, ec.value.msg) == (ei.value.code, ei.value.msg)
    return ei.value


def test_explain():
    plan = PL.SortMergeJoinExec(PL.build_join_schema(LS, RS, PL.JOIN_LEFT), _leaf(LS, "l"), _leaf(RS, "r"),
                                [(E.Column("k"), E.Column("rk")), (E.Column("j"), E.Column("rj"))], [(True, True), (False, False)], PL.JOIN_LEFT)
    text = plan.explain()
    first = text.splitlines()[0]
    assert first.startswith("SortMergeJoin: join_type=Left, on=[(k@0, rk@0), (j@1, rj@1)], sort_options=[ASC NULLS FIRST, DESC NULLS LAST] schema=[k:int64?")
    assert "  [left]\n    FFIReader" in text and "  [right]\n    FFIReader" in text
    assert text.index("[left]") < text.index("[right]")


@pytest.mark.parametrize("jt,name", [(PL.JOIN_INNER, "Inner"), (PL.JOIN_LEFT, "Left"), (PL.JOIN_RIGHT, "Right"), (PL.JOIN_FULL, "Full"),
                                     (PL.JOIN_SEMI, "LeftSemi"), (PL.JOIN_ANTI, "LeftAnti"), (PL.JOIN_EXISTENCE, "Existence")])
def test_every_join_type_decodes(jt, name):
    plan = PL.SortMergeJoinExec(PL.build_join_schema(LS, RS, jt), _leaf(LS, "l"), _leaf(RS, "r"), [(E.Column("k"), E.Column("rk"))], [ASC_NF], jt)
    assert plan.explain().startswith(f"SortMergeJoin: join_type={name}, ")


def test_a_sorted_right_subtree_decodes():
    right = PL.SortExec(_leaf(RS, "r"), [(E.Column("rk"), False, True)])
    left = PL.SortExec(_leaf(LS, "l"), [(E.Column("k"), False, True)])
    text = PL.SortMergeJoinExec(PL.build_join_schema(LS, RS, PL.JOIN_INNER), left, right, [(E.Column("k"), E.Column("rk"))], [ASC_NF], PL.JOIN_INNER).explain()
    assert "[left]\n    SortExec [k@0 ASC NULLS FIRST]" in text and "[right]\n    SortExec [rk@0 ASC NULLS FIRST]" in text


@pytest.mark.parametrize("missing", ["schema", "left", "right"])
def test_missing_fields(missing):
    n = _node([(E.Column("k"), E.Column("rk"))], [ASC_NF])
    n.sort_merge_join.ClearField(missing)
    e = _err(n)
    assert e.code == native.ERR_INVALID_PLAN and "Missing required field" in e.msg


@pytest.mark.parametrize("opts", [[], [ASC_NF, ASC_NF]])
def test_sort_options_count(opts):
    e = _err(_node([(E.Column("k"), E.Column("rk"))], opts))
    assert e.code == native.ERR_INVALID_PLAN and f"{len(opts)} sort_options for 1 join keys" in e.msg


def test_key_type_mismatch():
    e = _err(_node([(E.Column("k"), E.Column("rj"))], [ASC_NF]))
    assert e.code == native.ERR_INVALID_PLAN and "join key data type differs int64 <-> int32" in e.msg


def test_bad_join_type():
    n = _node([(E.Column("k"), E.Column("rk"))], [ASC_NF])
    n.sort_merge_join.join_type = 7
    e = _err(n)
    assert e.code == native.ERR_INVALID_PLAN and "invalid JoinType" in e.msg


def test_no_keys():
    e = _err(_node([], []))
    assert e.code == native.ERR_INVALID_PLAN and "join without keys" in e.msg


def test_three_keys():
    ls = Schema([Field("a", T.int32), Field("b", T.int32), Field("c", T.int32)])
    on = [(E.Column(x), E.Column(x)) for x in "abc"]
    e = _err(_node(on, [ASC_NF] * 3, ls=ls, rs=ls))
    assert e.code == native.ERR_UNSUPPORTED and "more than two join keys" in e.msg


def test_computed_key():
    on = [(E.BinaryExpr(E.Column("k"), "Plus", E.Literal(1, T.int64)), E.Column("rk"))]
    e = _err(_node(on, [ASC_NF]))
    assert e.code == native.ERR_UNSUPPORTED and "computed expression" in e.msg


@pytest.mark.parametrize("t", [T.utf8, T.float64, T.decimal128(20, 2), T.bool_])
def test_key_types_off_the_gpu_path(t):
    s = Schema([Field("x", t), Field("v", T.int64)])
    e = _err(_node([(E.Column("x"), E.Column("x"))], [ASC_NF], ls=s, rs=s))
    assert e.code == native.ERR_UNSUPPORTED and f"join key of type {t}" in e.msg


@pytest.mark.parametrize("side", ["left", "right"])
def test_string_data_column(side):
    s = Schema([Field("k", T.int64), Field("s", T.utf8)])
    ls, rs = (s, RS) if side == "left" else (LS, Schema([Field("rk", T.int64), Field("s", T.utf8)]))
    e = _err(_node([(E.Column("k"), E.Column("rk"))], [ASC_NF], ls=ls, rs=rs))
    assert e.code == native.ERR_UNSUPPORTED and "utf8 column in a join input" in e.msg


def test_output_schema_is_checked():
    bad = Schema(list(LS) + [Field("rk", T.int32, True)])
    e = _err(_node([(E.Column("k"), E.Column("rk"))], [ASC_NF], schema=bad))
    assert e.code == native.ERR_INVALID_PLAN and "join schema has 4 fields, the join produces 6" in e.msg
    e = _err(_node([(E.Column("k"), E.Column("rk"))], [ASC_NF], jt=PL.JOIN_EXISTENCE, schema=Schema(list(LS) + [Field("e", T.int8, False)])))
    assert e.code == native.ERR_INVALID_PLAN and "join schema field 3 is int8, the inputs give bool" in e.msg


def test_plan_class_validates_at_construction():
    with pytest.raises(native.NativeError) as ei:
        PL.SortMergeJoinExec(PL.build_join_schema(LS, RS, PL.JOIN_INNER), _leaf(LS, "l"), _leaf(RS, "r"), [(E.Column("k"), E.Column("rj"))], [ASC_NF], PL.JOIN_INNER)
    assert ei.value.code == native.ERR_INVALID_PLAN
