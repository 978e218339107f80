"""IpcReaderExecNode of blaze_b200/proto.py against the reference's field table for it (tests/golden/auron_proto_ipc_reader_fields.json,
auron.proto:31,607-611), and the PhysicalPlanNode oneof entry that carries it.  The mirror declares it nested in PhysicalPlanNode: only
the qualified name differs, not a byte on the wire."""
import json
import os

from google.protobuf import descriptor_pb2 as dpb

from blaze_b200 import proto as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "auron_proto_ipc_reader_fields.json")
F = dpb.FieldDescriptorProto
SCALAR = {F.TYPE_STRING: "string", F.TYPE_UINT32: "uint32"}


def test_ipc_reader_message_matches_reference_fields():
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
    entry, number = ref["plan_node_field"]
    field = next(f for f in pp.field if f.name == entry)
    assert field.number == number and field.type_name.split(".")[-1] == "IpcReaderExecNode"
