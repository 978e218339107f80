"""Spark runtime bloom filters without a GPU: the oracle against the reference's known answers, decode and explain of
XxHash64 / BloomFilterMightContain / the scalar-subquery wrapper through b200q_plan_explain, every refusal and validation
error, and the resolver protocol (op create resolves the scalar subquery before it looks for a device)."""
import json
import os
import struct

import numpy as np
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from blaze_b200.types import Field, Schema
from oracle import bloom_oracle as B

HERE = os.path.dirname(os.path.abspath(__file__))
KATS = json.load(open(os.path.join(HERE, "golden", "bloom_kats.json")))
S = Schema([Field("k", T.int64, True), Field("i", T.int32, True), Field("s", T.utf8, True), Field("b", T.bool_, True),
            Field("d", T.date32, True), Field("f", T.float64, True), Field("x", T.decimal128(10, 2), True), Field("y", T.binary, True)])


def filter_bytes(values, num_bits=1024, k=3):
    bf = B.SparkBloomFilter(k, B.SparkBitArray.with_num_bits(num_bits))
    for v in values:
        bf.put_long(v)
    return bf.write_to()


def bin_lit(b):
    return E.Literal(b, T.binary)


def might(value, flt, uuid="u1"):
    return E.BloomFilterMightContain(flt, value, uuid)


# ---- the oracle against the reference's vectors -------------------------------------------------------------------
def test_oracle_xxhash64_kats():
    for key, tn in (("xxhash64_int64", "int64"), ("xxhash64_utf8", "utf8")):
        assert B.spark_xxhash64([KATS[key]["values"]], [tn]) == KATS[key]["expected"]
    g = KATS["xxhash64_bytes_seed42"]
    assert [B.xxhash64(s.encode(), 42) for s in g["values"]] == g["expected"]


def test_oracle_hash_long_and_bit_array():
    g = KATS["murmur3_int64_seed42"]
    assert [B.hash_long(v, 42) for v in g["values"]] == g["expected"]
    g = KATS["bit_array_bit_size"]
    assert [B.SparkBitArray.with_num_bits(n).bit_size() for n in g["num_bits"]] == g["expected"]
    for bad in (0, 1 << 31):
        with pytest.raises(ValueError):
            B.SparkBitArray.with_num_bits(bad)
    rng = np.random.default_rng(37)                       # BitArraySuite: set / get and merge
    a, b = B.SparkBitArray.with_num_bits(320), B.SparkBitArray.with_num_bits(320)
    ia, ib = set(rng.integers(0, 320, 100).tolist()), set(rng.integers(0, 320, 100).tolist())
    for i in ia:
        a.set(i)
    for i in ib:
        b.set(i)
    assert all(a.get(i) for i in ia) and a.true_count() == len(ia)
    a.put_all(b)
    assert all(a.get(i) for i in ia | ib) and a.true_count() == len(ia | ib)


def test_oracle_bloom_filter_properties():
    """the bloom filter has no known answers in the reference: no false negatives, the bytes round-trip, optimal k and the
    shrink keep every inserted key"""
    rng = np.random.default_rng(5)
    keys = rng.integers(-2**63, 2**63 - 1, 2000, dtype=np.int64).tolist() + [0, -1, 2**63 - 1, -2**63]
    k = B.SparkBloomFilter.optimal_num_of_hash_functions(len(keys), 1 << 16)
    assert k == round((1 << 16) / len(keys) * np.log(2)) and B.SparkBloomFilter.optimal_num_of_hash_functions(10**6, 64) == 1
    bf = B.SparkBloomFilter(k, B.SparkBitArray.with_num_bits(1 << 16))
    for v in keys:
        bf.put_long(v)
    assert all(bf.might_contain_long(v) for v in keys)
    data = bf.write_to()
    assert len(data) == 12 + 8 * 1024 and B.SparkBloomFilter.read_from(data).write_to() == data
    sparse = B.SparkBloomFilter(3, B.SparkBitArray.with_num_bits(1 << 16))
    for v in keys[:10]:
        sparse.put_long(v)
    trues = sparse.bits.true_count()
    sparse.shrink_to_fit()
    assert 3 * trues * 2 <= sparse.bits.bit_size() < 3 * trues * 4 and all(sparse.might_contain_long(v) for v in keys[:10])
    assert B.might_contain(None, [1, None]) == [False, False] and B.might_contain(data, [keys[0], None]) == [True, None]


# ---- decode and explain ---------------------------------------------------------------------------------------------
def test_explain_xxhash64_and_might_contain_literal():
    data = filter_bytes([1, 2, 3], 1024, 3)
    plan = PL.FilterExec([might(E.XxHash64(E.Column("k"), E.Column("s")), bin_lit(data), "rf-7")], PL.MemoryExec(S))
    txt = plan.explain()
    assert "BloomFilterMightContain(uuid=rf-7, SparkBloomFilter(k=3, bits=1024), XxHash64(k@0, s@2))" in txt
    null = PL.FilterExec([might(E.Column("i"), bin_lit(None))], PL.MemoryExec(S)).explain()
    assert "BloomFilterMightContain(uuid=u1, NULL:binary, i@1)" in null
    proj = PL.ProjectExec([(E.XxHash64(E.Column("b"), E.Column("d"), E.Literal(None, T.null)), "h")], PL.MemoryExec(S))
    assert proj.schema()[0].dtype == T.int64 and "XxHash64(b@3, d@4, NULL:null)" in proj.explain()


def test_explain_scalar_subquery_never_calls_the_resolver():
    calls = []
    native.set_scalar_subquery_resolver(lambda s: calls.append(s) or filter_bytes([1]))
    try:
        plan = PL.FilterExec([might(E.XxHash64(E.Column("k")), E.ScalarSubquery(b"\x01\x02\x03"))], PL.MemoryExec(S))
        assert "BloomFilterMightContain(uuid=u1, ScalarSubquery(3 bytes), XxHash64(k@0))" in plan.explain()
        assert calls == []
    finally:
        native.set_scalar_subquery_resolver(None)


@pytest.mark.parametrize("col", ["f", "x", "y"])
def test_xxhash64_of_float_decimal_binary_is_unsupported(col):
    with pytest.raises(native.NativeError) as ei:
        PL.ProjectExec([(E.XxHash64(E.Column(col)), "h")], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED and "XxHash64 over a" in ei.value.msg


def test_xxhash64_must_return_int64():
    with pytest.raises(native.NativeError) as ei:
        PL.ProjectExec([(E.ScalarFunction("XxHash64", [E.Column("k")], T.int32), "h")], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_INVALID_PLAN and "XxHash64 must return int64" in ei.value.msg


@pytest.mark.parametrize("col", ["s", "y", "f", "d", "b"])
def test_might_contain_value_types_outside_int8_int64_are_unsupported(col):
    with pytest.raises(native.NativeError) as ei:
        PL.FilterExec([might(E.Column(col), bin_lit(filter_bytes([1])))], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED and "BloomFilterMightContain over a" in ei.value.msg


def test_filter_argument_must_be_binary_literal_or_subquery():
    with pytest.raises(native.NativeError) as ei:
        PL.FilterExec([might(E.Column("k"), E.Column("y"))], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED and "only a Binary literal or a scalar subquery" in ei.value.msg
    with pytest.raises(native.NativeError) as ei:
        PL.FilterExec([might(E.Column("k"), E.Literal("abc", T.utf8))], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_INVALID_PLAN and "must be a Binary value" in ei.value.msg
    with pytest.raises(native.NativeError) as ei:
        PL.FilterExec([might(E.Column("k"), E.ScalarSubquery(b"x", T.int64))], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_INVALID_PLAN and "scalar subquery must return Binary" in ei.value.msg


def test_subquery_wrapper_and_binary_literal_stay_refused_elsewhere():
    with pytest.raises(native.NativeError) as ei:
        PL.ProjectExec([(E.ScalarSubquery(b"x", T.int64), "v")], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED and "scalar subquery wrappers" in ei.value.msg
    with pytest.raises(native.NativeError) as ei:
        PL.FilterExec([E.IsNull(bin_lit(b"abc"))], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_UNSUPPORTED and "binary literals are not on the hot path" in ei.value.msg


def _header(version=1, k=3, words=2):
    return struct.pack(">iii", version, k, words)


MALFORMED = {
    "version": (_header(version=2) + bytes(16), "unsupported version 2"),
    "k_zero": (_header(k=0) + bytes(16), "num_hash_functions 0 is not positive"),
    "k_negative": (_header(k=-4) + bytes(16), "num_hash_functions -4 is not positive"),
    "words_zero": (_header(words=0), "num_words 0 is not positive"),
    "words_negative": (_header(words=-1), "num_words -1 is not positive"),
    "too_many_bits": (_header(words=1 << 25), "more than INT32_MAX bits"),
    "truncated_header": (_header()[:11], "shorter than the 12-byte header"),
    "truncated_words": (_header() + bytes(15), "27 bytes where num_words 2 needs 28"),
    "extra_bytes": (_header() + bytes(17), "29 bytes where num_words 2 needs 28"),
    "empty": (b"", "0 bytes, shorter than the 12-byte header"),
}


@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_malformed_literal_filters_are_invalid_arg(case):
    data, msg = MALFORMED[case]
    with pytest.raises(native.NativeError) as ei:
        PL.FilterExec([might(E.Column("k"), bin_lit(data))], PL.MemoryExec(S))
    assert ei.value.code == native.ERR_INVALID_ARG and msg in ei.value.msg, ei.value.msg


# ---- the resolver, at op create ---------------------------------------------------------------------------------------
def _create(plan):
    return native.NativeOp(plan.plan_bytes())


def _subquery_plan(n=1):
    preds = [might(E.XxHash64(E.Column("k")), E.ScalarSubquery(bytes([i])), f"u{i}") for i in range(n)]
    return PL.FilterExec(preds, PL.MemoryExec(S))


def test_missing_resolver_is_unsupported():
    native.set_scalar_subquery_resolver(None)
    with pytest.raises(native.NativeError) as ei:
        _create(_subquery_plan())
    assert ei.value.code == native.ERR_UNSUPPORTED and "scalar subquery needs a resolver" in ei.value.msg


@pytest.mark.parametrize("case", ["version", "k_zero", "truncated_words", "extra_bytes"])
def test_malformed_resolved_filters_are_invalid_arg(case):
    data, msg = MALFORMED[case]
    calls = []
    native.set_scalar_subquery_resolver(lambda s: calls.append(s) or data)
    try:
        with pytest.raises(native.NativeError) as ei:
            _create(_subquery_plan())
        assert ei.value.code == native.ERR_INVALID_ARG and msg in ei.value.msg
        assert calls == [b"\x00"]
    finally:
        native.set_scalar_subquery_resolver(None)


def test_resolver_failure_is_an_execution_error_and_calls_are_one_per_expression():
    calls = []

    def fail(s):
        calls.append(s)
        raise RuntimeError("subquery failed")
    native.set_scalar_subquery_resolver(fail)
    try:
        with pytest.raises(native.NativeError) as ei:
            _create(_subquery_plan(3))
        assert ei.value.code == native.ERR_EXECUTION and "resolver failed" in ei.value.msg
        assert calls == [b"\x00"]                       # the first failure stops the create
        calls.clear()
        native.set_scalar_subquery_resolver(lambda s: calls.append(s) or filter_bytes([int(s[0])]))
        try:
            _create(_subquery_plan(3)).close()
        except native.NativeError as e:                 # without a GPU the create stops at the device check, after resolving
            assert e.code == native.ERR_NO_DEVICE
        assert calls == [b"\x00", b"\x01", b"\x02"]
    finally:
        native.set_scalar_subquery_resolver(None)


def test_symbol_is_exported():
    assert "b200q_set_scalar_subquery_resolver" in native.SYMBOLS


def test_proto_messages_match_reference_fields():
    """the mirror nests both messages in PhysicalExprNode: only the qualified names differ, not a byte on the wire"""
    from google.protobuf import descriptor_pb2 as dpb
    from blaze_b200 import proto as P
    F = dpb.FieldDescriptorProto
    scalar = {F.TYPE_BOOL: "bool", F.TYPE_BYTES: "bytes", F.TYPE_STRING: "string"}
    ref = json.load(open(os.path.join(HERE, "golden", "auron_proto_bloom_fields.json")))
    px = next(m for m in P.FILE_DESCRIPTOR.message_type if m.name == "PhysicalExprNode")
    nested = {m.name: m for m in px.nested_type}
    for name, fields in ref["messages"].items():
        m = nested[name]
        assert {f.name for f in m.field} == set(fields)
        for f in m.field:
            num, typ, rep = fields[f.name]
            ours = f.type_name.split(".")[-1] if f.type in (F.TYPE_MESSAGE, F.TYPE_ENUM) else scalar[f.type]
            assert (f.number, ours, f.label == F.LABEL_REPEATED) == (num, typ, rep), f"{name}.{f.name}"
    for entry, number in ref["expr_node_fields"].items():
        field = next(f for f in px.field if f.name == entry)
        assert field.number == number and px.oneof_decl[field.oneof_index].name == "ExprType"


# ---- BLOOM_FILTER aggregate: decode, explain and refusals ---------------------------------------------------------------
def _bloom_agg_plan(child=None, est=1000, nbits=8192, groupings=(), extra=()):
    ch = [child if child is not None else E.XxHash64(E.Column("k")), E.Literal(est, T.int64), E.Literal(nbits, T.int64)]
    aggs = [E.AggExpr("bf", E.PARTIAL, PL.create_agg(E.AGG_BLOOM_FILTER, ch, S, T.binary))] + list(extra)
    return PL.AggExec(PL.HashAgg, list(groupings), aggs, False, PL.MemoryExec(S))


def test_bloom_agg_explain_and_optimal_k():
    txt = _bloom_agg_plan(est=1000, nbits=8192).explain()
    k = B.SparkBloomFilter.optimal_num_of_hash_functions(1000, 8192)
    assert f"BloomFilter(XxHash64(k@0))[num_bits=8192, k={k}]:binary/Partial AS bf" in txt and "schema=[#9223372036854775807:binary]" in txt
    assert "k=1]" in _bloom_agg_plan(est=10**9, nbits=64).explain()


@pytest.mark.parametrize("nbits", [3, 1000, 0, -64])
def test_bloom_agg_num_bits_must_be_a_power_of_two(nbits):
    with pytest.raises(native.NativeError) as ei:
        _bloom_agg_plan(nbits=nbits)
    assert ei.value.code == native.ERR_INVALID_PLAN and "is not a power of two" in ei.value.msg


def test_bloom_agg_refusals():
    with pytest.raises(native.NativeError) as ei:
        _bloom_agg_plan(groupings=[E.GroupingExpr("i", E.Column("i"))])
    assert ei.value.code == native.ERR_UNSUPPORTED and "with grouping keys" in ei.value.msg
    with pytest.raises(native.NativeError) as ei:
        _bloom_agg_plan(extra=[E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Column("k")], S, T.int64))])
    assert ei.value.code == native.ERR_UNSUPPORTED and "next to other aggregates" in ei.value.msg
    for c in ("s", "y", "f"):
        with pytest.raises(native.NativeError) as ei:
            _bloom_agg_plan(child=E.Column(c))
        assert ei.value.code == native.ERR_UNSUPPORTED and "BLOOM_FILTER over a" in ei.value.msg
    with pytest.raises(native.NativeError) as ei:
        _bloom_agg_plan(est=0)
    assert ei.value.code == native.ERR_INVALID_PLAN and "estimated_num_items 0" in ei.value.msg


def test_oracle_frozen_row_and_final_bytes():
    assert B.frozen_row(None) == b"\x00" and B.final_bytes(None) is None
    bf = B.bloom_agg([[], [1, None, 2]], 100, 1024)
    assert bf.k == B.SparkBloomFilter.optimal_num_of_hash_functions(100, 1024)
    assert B.frozen_row(bf) == b"\x01" + bf.write_to() and B.bloom_agg([[]], 100, 1024) is None
    shrunk = B.SparkBloomFilter.read_from(B.final_bytes(bf))
    assert shrunk.bits.bit_size() < 1024 and shrunk.might_contain_long(1) and shrunk.might_contain_long(2)
