"""ExpandExecNode / ExpandProjection of blaze_b200/proto.py against the reference's field table for them
(tests/golden/auron_proto_expand_fields.json, auron.proto:714-722), and the PhysicalPlanNode oneof entry that carries them.
The mirror declares the two messages nested in PhysicalPlanNode: only the qualified name differs, not a byte on the wire."""
import json
import os

from google.protobuf import descriptor_pb2 as dpb

from blaze_b200 import exprs as E, plans as PL, proto as P, types as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "auron_proto_expand_fields.json")
F = dpb.FieldDescriptorProto


def test_expand_messages_match_reference_fields():
    ref = json.load(open(GOLDEN))["messages"]
    pp = next(m for m in P.FILE_DESCRIPTOR.message_type if m.name == "PhysicalPlanNode")
    nested = {m.name: m for m in pp.nested_type}
    assert set(ref) <= set(nested)
    for name, fields in ref.items():
        m = nested[name]
        assert {f.name for f in m.field} == set(fields)
        for f in m.field:
            num, typ, rep = fields[f.name]
            assert f.number == num and (f.label == F.LABEL_REPEATED) == rep and f.type == F.TYPE_MESSAGE
            assert f.type_name.split(".")[-1] == typ
    expand = next(f for f in pp.field if f.name == "expand")
    assert expand.number == 20 and expand.type_name.split(".")[-1] == "ExpandExecNode"


def test_expand_node_wire_bytes():
    """tag 20 (wire type 2) of PhysicalPlanNode, then input = 1, schema = 2, one projections = 3 entry per projection"""
    s = T.Schema([T.Field("a", T.int64, False)])
    leaf = PL.MemoryExec(s)
    node = P.PhysicalPlanNode()
    node.ParseFromString(PL.ExpandExec(s, [[E.Column("a")], [E.Literal(1, T.int64)]], leaf).plan_bytes())
    assert node.WhichOneof("PhysicalPlanType") == "expand"
    assert len(node.expand.projections) == 2 and node.expand.input.WhichOneof("PhysicalPlanType") == "ffi_reader"
    b = node.SerializeToString()
    assert b[:2] == b"\xa2\x01"                                         # varint of (20 << 3) | 2
    inner = node.expand.SerializeToString()
    assert inner[0] == (1 << 3) | 2
