"""ExpandExec test material shared by the oracle, host and GPU tests: the reference's KATs (tests/golden/expand_kats.json) as plans,
and ROLLUP / CUBE / GROUPING SETS projections built the way Spark's Expand does (every grouping column is either carried or a typed
NULL in a set, the grouping id is a literal)."""
import json
import os

import numpy as np
import pyarrow as pa

from blaze_b200 import exprs as E, types as T
from blaze_b200.types import Field, Schema

HERE = os.path.dirname(os.path.abspath(__file__))
KATS = json.load(open(os.path.join(HERE, "golden", "expand_kats.json")))["cases"]

_TYPES = {"int32": (T.int32, pa.int32(), np.int32), "float32": (T.float32, pa.float32(), np.float32), "bool": (T.bool_, pa.bool_(), bool)}


def kat_input(case):
    """-> (schema, record batch) of the KAT's one non-nullable input column"""
    dt, pt, npt = _TYPES[case["type"]]
    vals = [npt(float(v)) if case["type"] == "float32" else v for v in case["input"]]
    rb = pa.RecordBatch.from_arrays([pa.array(vals, type=pt)], schema=pa.schema([pa.field(case["column"], pt, nullable=False)]))
    return Schema([Field(case["column"], dt, False)]), rb


def kat_projections(case):
    dt = _TYPES[case["type"]][0]
    out = []
    for op, lit in case["projections"]:
        v = np.float32(float(lit)).item() if case["type"] == "float32" else lit
        out.append([E.BinaryExpr(E.Column(case["column"]), op, E.Literal(v, dt))])
    return out


def kat_text(case, values):
    """values of one output column in the KAT's notation (float32: shortest round-trip text, -0.0 kept)"""
    if case["type"] == "float32":
        return [str(np.float32(v)) for v in values]
    return list(values)


def grouping_sets(kind, nkeys):
    """the sets of ROLLUP / CUBE over keys 0..nkeys-1, as tuples of the grouped key indices, in Spark's order"""
    if kind == "rollup":
        return [tuple(range(i)) for i in range(nkeys, -1, -1)]
    if kind == "cube":
        return [tuple(k for k in range(nkeys) if not (m >> (nkeys - 1 - k)) & 1) for m in range(1 << nkeys)]
    raise ValueError(kind)


def grouping_id(grouped, nkeys):
    """Spark's grouping id: bit (nkeys - 1 - k) set when key k is rolled up"""
    return sum(1 << (nkeys - 1 - k) for k in range(nkeys) if k not in grouped)


def expand_for_sets(in_schema: Schema, keys, carried, sets, gid_type=T.int64):
    """-> (expand output schema, projections): the key columns (NULL when rolled up), the carried columns, then `spark_grouping_id`"""
    nk = len(keys)
    fields = [Field(k, in_schema[in_schema.index_of(k)].dtype, True) for k in keys]
    fields += [in_schema[in_schema.index_of(c)] for c in carried]
    fields.append(Field("spark_grouping_id", gid_type, False))
    projs = []
    for g in sets:
        p = [E.Column(k) if i in g else E.Literal(None, fields[i].dtype) for i, k in enumerate(keys)]
        p += [E.Column(c) for c in carried]
        p.append(E.Literal(grouping_id(g, nk), gid_type))
        projs.append(p)
    return Schema(fields), projs
