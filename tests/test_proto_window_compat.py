"""WindowExecNode / WindowExprNode / WindowGroupLimit and the WindowFunction / WindowFunctionType enums of blaze_b200/proto.py against
the reference's field table for them (tests/golden/auron_proto_window_fields.json, auron.proto:121-125, 537-562), and the
PhysicalPlanNode oneof entry that carries them.  The mirror declares them nested in PhysicalPlanNode: only the qualified names
differ, not a byte on the wire."""
import json
import os

from google.protobuf import descriptor_pb2 as dpb

from blaze_b200 import exprs as E, plans as PL, proto as P, types as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "auron_proto_window_fields.json")
F = dpb.FieldDescriptorProto
SCALAR = {F.TYPE_BOOL: "bool", F.TYPE_UINT32: "uint32"}


def test_window_messages_match_reference_fields():
    ref = json.load(open(GOLDEN))
    pp = next(m for m in P.FILE_DESCRIPTOR.message_type if m.name == "PhysicalPlanNode")
    nested = {m.name: m for m in pp.nested_type}
    for name, fields in ref["messages"].items():
        m = nested[name]
        assert {f.name for f in m.field} == set(fields)
        for f in m.field:
            num, typ, rep = fields[f.name]
            ours = f.type_name.split(".")[-1] if f.type in (F.TYPE_MESSAGE, F.TYPE_ENUM) else SCALAR[f.type]
            assert (f.number, ours, f.label == F.LABEL_REPEATED) == (num, typ, rep), f"{name}.{f.name}"
    enums = {e.name: {v.name: v.number for v in e.value} for e in pp.enum_type}
    assert {k: enums[k] for k in ref["enums"]} == ref["enums"]
    window = next(f for f in pp.field if f.name == "window")
    assert window.number == 22 and window.type_name.split(".")[-1] == "WindowExecNode"


def test_window_node_wire_bytes():
    """tag 22 (wire type 2) of PhysicalPlanNode; return_type = 1000 of WindowExprNode; k of the group limit; the order spec as
    PhysicalExprNode.sort entries"""
    s = T.Schema([T.Field("a", T.int64, False), T.Field("b", T.int64, False)])
    w = PL.WindowExec(PL.MemoryExec(s), [E.WindowExpr.rank_like("rk", E.RANK)], [E.Column("a")], [(E.Column("b"), True, False)], 7, False)
    node = P.PhysicalPlanNode()
    node.ParseFromString(w.plan_bytes())
    assert node.WhichOneof("PhysicalPlanType") == "window"
    wn = node.window
    assert wn.group_limit.k == 7 and not wn.output_window_cols and wn.window_expr[0].window_func == E.RANK
    assert wn.order_spec[0].WhichOneof("ExprType") == "sort" and not wn.order_spec[0].sort.asc
    assert node.SerializeToString()[:2] == b"\xb2\x01"                  # varint of (22 << 3) | 2
    x = wn.window_expr[0].SerializeToString()
    assert b"\xc2\x3e" in x                                              # varint of (1000 << 3) | 2: return_type
