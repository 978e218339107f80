"""SortMergeJoinExecNode and SortOptions of blaze_b200/proto.py against the reference's field table for them
(tests/golden/auron_proto_smj_fields.json, auron.proto:38,432-439,485-488), and the PhysicalPlanNode oneof entry that carries the
node.  The mirror declares both nested in PhysicalPlanNode: only the qualified names differ, not a byte on the wire."""
import json
import os

from google.protobuf import descriptor_pb2 as dpb

from blaze_b200 import proto as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "auron_proto_smj_fields.json")
F = dpb.FieldDescriptorProto
SCALAR = {F.TYPE_BOOL: "bool"}


def test_smj_messages_match_reference_fields():
    ref = json.load(open(GOLDEN))
    pp = next(m for m in P.FILE_DESCRIPTOR.message_type if m.name == "PhysicalPlanNode")
    nested = {m.name: m for m in pp.nested_type}
    assert set(ref["messages"]) == {"SortMergeJoinExecNode", "SortOptions"}
    for name, fields in ref["messages"].items():
        m = nested[name]
        assert {f.name for f in m.field} == set(fields)
        for f in m.field:
            num, typ, rep = fields[f.name]
            ours = f.type_name.split(".")[-1] if f.type in (F.TYPE_MESSAGE, F.TYPE_ENUM) else SCALAR[f.type]
            assert (f.number, ours, f.label == F.LABEL_REPEATED) == (num, typ, rep), f"{name}.{f.name}"


def test_sort_merge_join_oneof_entry():
    ref = json.load(open(GOLDEN))
    pp = next(m for m in P.FILE_DESCRIPTOR.message_type if m.name == "PhysicalPlanNode")
    entry, number = ref["plan_node_field"]
    field = next(f for f in pp.field if f.name == entry)
    assert field.number == number == 10 and field.type_name.split(".")[-1] == "SortMergeJoinExecNode"
    assert field.HasField("oneof_index") and pp.oneof_decl[field.oneof_index].name == "PhysicalPlanType"


def test_smj_node_round_trips_on_the_wire():
    from blaze_b200 import exprs as E, types as T
    from blaze_b200.types import Field, Schema
    s = Schema([Field("k", T.int64, True)])
    n = P.smj_node(Schema([Field("k", T.int64, True), Field("k", T.int64, True)]), P.ffi_reader_node(s, "l"), P.ffi_reader_node(s, "r"),
                   [(E.Column("k"), E.Column("k"))], [(False, True)], 2)
    back = P.PhysicalPlanNode.FromString(n.SerializeToString())
    assert back.WhichOneof("PhysicalPlanType") == "sort_merge_join"
    j = back.sort_merge_join
    assert j.join_type == 2 and [(o.asc, o.nulls_first) for o in j.sort_options] == [(False, True)] and len(j.on) == 1
