"""Spark runtime bloom filters on the GPU, through the C ABI, against oracle/bloom_oracle.py: XxHash64 bit for bit through
ProjectExec, BloomFilterMightContain row for row through ProjectExec and FilterExec (host and device batches, several batch
splits, k from 1 to 30, 64 bits to 2^26 bits, a NULL filter, NULL values), Filter(might_contain(XxHash64(k))) -> AggExec
Partial -> Final fused and as two ops, a filter handed over by a scalar-subquery resolver, and the kernel choice.  The
BLOOM_FILTER aggregate byte for byte against the oracle: Partial / PartialMerge / Final / fused, frozen-row and columnar state,
through ShuffleWriterExec -> IpcReaderExec, both None cases, and a GPU-built filter feeding might_contain."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from oracle import bloom_oracle as B

pytestmark = pytest.mark.gpu

I64_EDGES = [0, 1, -1, 2**63 - 1, -2**63, 2**31 - 1, -2**31, 2**32, 42]


def build_filter(keys, num_bits, k):
    bf = B.SparkBloomFilter(k, B.SparkBitArray.with_num_bits(num_bits))
    for v in keys:
        bf.put_long(int(v))
    return bf.write_to()


def batches_of(rb, rows):
    return [rb.slice(i, rows) for i in range(0, rb.num_rows, rows)]


def project(rb, exprs, batch_rows=10_000, conf=None):
    batches = batches_of(rb, batch_rows)
    plan = PL.ProjectExec(exprs, PL.MemoryExec.from_arrow(batches, rb.schema))
    got = PL.collect(plan, conf)
    return pa.Table.from_batches(got, schema=got[0].schema) if got else None, plan


def col(rb, name):
    return rb.column(rb.schema.get_field_index(name)).to_pylist()


# ---- XxHash64 -------------------------------------------------------------------------------------------------------
def typed_table(n, seed, null_frac=0.15):
    rng = np.random.default_rng(seed)
    m = lambda: rng.random(n) < null_frac
    i64 = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    i64[: len(I64_EDGES)] = I64_EDGES
    strs = ["", "a", "hello", "bar", "😁", "天地", "x" * 31, "y" * 32, "z" * 33, "abcdefghijklmnopqrstuvwxyz0123456789" * 3]
    return pa.RecordBatch.from_arrays([
        pa.array(rng.random(n) < 0.5, mask=m()),
        pa.array(rng.integers(-128, 128, n, dtype=np.int8), mask=m()),
        pa.array(rng.integers(-2**15, 2**15, n, dtype=np.int16), mask=m()),
        pa.array(rng.integers(-2**31, 2**31, n, dtype=np.int32), mask=m()),
        pa.array(i64, mask=m()),
        pa.array(rng.integers(-10**6, 10**6, n, dtype=np.int32), type=pa.int32(), mask=m()).cast(pa.date32()),
        pa.array(rng.integers(-2**62, 2**62, n, dtype=np.int64), mask=m()).cast(pa.timestamp("us")),
        pa.array([strs[i % len(strs)] + str(i % 7) * (i % 5) for i in range(n)], mask=m()),
    ], names=["b", "i8", "i16", "i32", "i64", "d", "ts", "s"])


TYPE_NAMES = {"b": "bool", "i8": "int8", "i16": "int16", "i32": "int32", "i64": "int64", "d": "date32", "ts": "timestamp[us]", "s": "utf8"}


def _pyvals(rb, name):
    """the column as Python ints (dates as days, timestamps as microseconds: most of them lie outside datetime's range)"""
    c = rb.column(rb.schema.get_field_index(name))
    if name == "d":
        return c.view(pa.int32()).to_pylist()
    if name == "ts":
        return c.view(pa.int64()).to_pylist()
    return c.to_pylist()


def test_xxhash64_reference_vectors():
    rb = pa.RecordBatch.from_arrays([pa.array([1, 0, -1, 2**63 - 1, -2**63], pa.int64()), pa.array(["hello", "bar", "", "😁", "天地"])],
                                    names=["l", "s"])
    got, _ = project(rb, [(E.XxHash64(E.Column("l")), "hl"), (E.XxHash64(E.Column("s")), "hs")])
    assert got.column("hl").to_pylist() == [-7001672635703045582, -5252525462095825812, 3858142552250413010, -3246596055638297850, -8619748838626508300]
    assert got.column("hs").to_pylist() == [-4367754540140381902, -1798770879548125814, -7444071767201028348, -6337236088984028203, -235771157374669727]


@pytest.mark.parametrize("children", [["b"], ["i8"], ["i16"], ["i32"], ["i64"], ["d"], ["ts"], ["s"],
                                      ["i64", "s", "b"], ["b", "i8", "i16", "i32", "i64", "d", "ts", "s"]])
def test_xxhash64_every_type_with_nulls(children):
    rb = typed_table(20_000, seed=len(children) * 7 + len(children[0]))
    got, _ = project(rb, [(E.XxHash64(*[E.Column(c) for c in children]), "h")], batch_rows=7_001)
    exp = B.spark_xxhash64([_pyvals(rb, c) for c in children], [TYPE_NAMES[c] for c in children])
    assert got.column("h").null_count == 0 and got.column("h").to_pylist() == exp


def test_xxhash64_with_literal_and_null_children():
    rb = typed_table(5_000, seed=3)
    e = E.XxHash64(E.Literal(7, T.int32), E.Column("i64"), E.Literal(None, T.int64), E.Literal("k", T.utf8))
    got, _ = project(rb, [(e, "h")])
    n = rb.num_rows
    exp = B.spark_xxhash64([[7] * n, _pyvals(rb, "i64"), [None] * n, ["k"] * n], ["int32", "int64", "int64", "utf8"])
    assert got.column("h").to_pylist() == exp


# ---- might_contain --------------------------------------------------------------------------------------------------
def probe_table(n, seed, keys, null_frac=0.1):
    """values: half drawn from the inserted keys, the rest random, plus the i64 extremes; NULLs"""
    rng = np.random.default_rng(seed)
    v = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    take = rng.random(n) < 0.5
    v[take] = np.asarray(keys, dtype=np.int64)[rng.integers(0, len(keys), int(take.sum()))]
    v[: len(I64_EDGES)] = I64_EDGES
    mask = rng.random(n) < null_frac
    mask[: len(I64_EDGES)] = False
    return pa.RecordBatch.from_arrays([pa.array(v, mask=mask), pa.array(np.arange(n, dtype=np.int64))], names=["v", "row"])


@pytest.mark.parametrize("num_bits,k", [(64, 1), (64, 30), (1024, 3), (4096, 7), (1 << 20, 5), (1 << 26, 30), (1 << 26, 2)])
def test_might_contain_row_for_row(num_bits, k):
    rng = np.random.default_rng(num_bits + k)
    keys = rng.integers(-2**63, 2**63 - 1, max(8, min(2000, num_bits // 16)), dtype=np.int64).tolist() + I64_EDGES[:4]
    data = build_filter(keys, num_bits, k)
    rb = probe_table(30_000, seed=k, keys=keys)
    got, _ = project(rb, [(E.BloomFilterMightContain(E.Literal(data, T.binary), E.Column("v"), "u"), "m"), (E.Column("row"), "row")],
                     batch_rows=9_999)
    exp = B.might_contain(data, col(rb, "v"))
    m, ks = got.column("m").to_pylist(), set(keys)
    assert m == exp
    assert all(x for x, v in zip(m, col(rb, "v")) if v in ks)                 # no false negatives


def test_might_contain_negative_combined_hashes_and_narrow_ints():
    """the values whose h1 + i * h2 goes negative for some i take the flip; Int8..Int32 values are probed as i64"""
    keys = list(range(-300, 300))
    data = build_filter(keys, 2048, 9)
    neg = [v for v in range(-5000, 5000) if any(B._i32(B.hash_long(v, 0) + i * B.hash_long(v, B.hash_long(v, 0))) < 0 for i in range(1, 10))]
    assert len(neg) > 1000
    rb = pa.RecordBatch.from_arrays([pa.array(np.array(neg[:4000], dtype=np.int16)), pa.array(np.array(neg[:4000], dtype=np.int32)),
                                     pa.array(np.array(neg[:4000], dtype=np.int64)), pa.array(np.array([v % 128 for v in neg[:4000]], dtype=np.int8))],
                                    names=["a", "b", "c", "d"])
    lit = E.Literal(data, T.binary)
    got, _ = project(rb, [(E.BloomFilterMightContain(lit, E.Column(c)), c) for c in "abcd"])
    for c in "abcd":
        assert got.column(c).to_pylist() == B.might_contain(data, col(rb, c)), c


def test_null_filter_is_false_and_null_values_are_null():
    rb = probe_table(10_000, seed=1, keys=[1, 2, 3], null_frac=0.3)
    data = build_filter([1, 2, 3], 64, 2)
    got, _ = project(rb, [(E.BloomFilterMightContain(E.Literal(None, T.binary), E.Column("v")), "n"),
                          (E.BloomFilterMightContain(E.Literal(data, T.binary), E.Column("v")), "m")])
    assert got.column("n").to_pylist() == [False] * rb.num_rows
    assert got.column("m").to_pylist() == B.might_contain(data, col(rb, "v"))
    assert got.column("m").null_count == rb.column(0).null_count


@pytest.mark.parametrize("rows", [1, 777, 4096, 100_000])
def test_filter_by_might_contain_xxhash64_across_splits(rows):
    rng = np.random.default_rng(rows)
    n = 100_000
    k = rng.integers(0, 50_000, n, dtype=np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(k, mask=rng.random(n) < 0.05), pa.array(np.arange(n, dtype=np.int64))], names=["k", "row"])
    build = list(range(0, 50_000, 10))
    data = build_filter([B.xxhash64(int(x).to_bytes(8, "little", signed=True), 42) for x in build], 1 << 16, 4)
    pred = E.BloomFilterMightContain(E.Literal(data, T.binary), E.XxHash64(E.Column("k")), "rf")
    batches = batches_of(rb, rows)
    got = PL.collect(PL.FilterExec([pred], PL.MemoryExec.from_arrow(batches, rb.schema)))
    got_rows = sorted(r for b in got for r in b.column(1).to_pylist())
    hk = B.spark_xxhash64([col(rb, "k")], ["int64"])
    m = B.might_contain(data, [None if v is None else h for v, h in zip(col(rb, "k"), hk)])
    assert got_rows == [i for i, x in enumerate(m) if x]
    assert set(i for i, v in enumerate(col(rb, "k")) if v is not None and v % 10 == 0) <= set(got_rows)   # no false negatives


def _device_batch(rb, torch):
    cols, keep = [], []
    for c in rb.columns:
        v = torch.tensor(c.fill_null(0).to_numpy(), device="cuda")
        valid = None
        if c.null_count:                                     # packed from the values: a slice's bitmap starts at its offset
            valid = torch.tensor(np.packbits(c.is_valid().to_numpy(zero_copy_only=False), bitorder="little"), device="cuda")
        cols.append((v.data_ptr(), valid.data_ptr() if valid is not None else 0, len(c)))
        keep += [v] + ([valid] if valid is not None else [])
    return native.DeviceBatch(cols, rb.num_rows, 0, keep)


def test_might_contain_on_device_batches():
    torch = pytest.importorskip("torch")
    keys = list(range(0, 1_000_000, 7))
    data = build_filter(keys, 1 << 22, 6)
    rb = probe_table(200_000, seed=9, keys=keys)
    plan = PL.ProjectExec([(E.BloomFilterMightContain(E.Literal(data, T.binary), E.Column("v")), "m"), (E.Column("row"), "row")],
                          PL.MemoryExec.from_arrow([rb], rb.schema))
    with native.NativeOp(plan.plan_bytes()) as op:
        for part in batches_of(rb, 65_536):
            op.push_device(_device_batch(part, torch))
        op.finish()
        got = op.pull_all()
    t = pa.Table.from_batches(got)
    assert t.column("row").to_pylist() == list(range(rb.num_rows))
    assert t.column("m").to_pylist() == B.might_contain(data, col(rb, "v"))


# ---- Filter(might_contain) -> AggExec ------------------------------------------------------------------------------
def _agg_case(n=200_000, seed=4):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 100_000, n, dtype=np.int64)
    g = rng.integers(0, 500, n, dtype=np.int64)
    v = rng.integers(-10**9, 10**9, n, dtype=np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(k), pa.array(g), pa.array(v, mask=rng.random(n) < 0.1)], names=["k", "g", "v"])
    build = rng.choice(100_000, 10_000, replace=False)
    data = build_filter([B.xxhash64(int(x).to_bytes(8, "little", signed=True), 42) for x in build], 1 << 17, 5)
    survive = B.might_contain(data, B.spark_xxhash64([k.tolist()], ["int64"]))
    exp = {}
    for kk, gg, vv, s in zip(k.tolist(), g.tolist(), col(rb, "v"), survive):
        if s:
            cur = exp.setdefault(gg, [None, 0])
            if vv is not None:
                cur[0] = (cur[0] or 0) + vv
                cur[1] += 1
    return rb, data, exp


def _agg_plans(rb, pred):
    leaf = PL.MemoryExec.from_arrow(batches_of(rb, 50_000), rb.schema)
    ins = leaf.schema()
    gk = [E.GroupingExpr("g", E.Column("g"))]
    mk = lambda mode, ch: [E.AggExpr("s", mode, PL.create_agg(E.AGG_SUM, ch, ins, T.int64)), E.AggExpr("c", mode, PL.create_agg(E.AGG_COUNT, ch, ins, T.int64))]
    partial = PL.AggExec(PL.HashAgg, gk, mk(E.PARTIAL, [E.Column("v")]), False, PL.FilterExec([pred], leaf))
    final = PL.AggExec(PL.HashAgg, gk, mk(E.FINAL, [E.placeholder(T.int64)]), False, partial)
    return partial, final


def _rows(batches):
    out = {}
    for b in batches:
        for g, s, c in zip(*(b.column(i).to_pylist() for i in range(3))):
            out[g] = [s, c]
    return out


@pytest.mark.parametrize("generic", [False, True])
def test_filter_might_contain_then_agg_fused(generic):
    rb, data, exp = _agg_case()
    pred = E.BloomFilterMightContain(E.Literal(data, T.binary), E.XxHash64(E.Column("k")), "rf")
    _, final = _agg_plans(rb, pred)
    got = PL.collect(final, native.default_conf(force_generic_kernels=int(generic)))
    assert _rows(got) == exp
    assert final.last_metrics["fast_path_launches"] == 0          # a program with bloom probes runs on the VM kernel


def test_filter_might_contain_then_agg_as_two_ops():
    rb, data, exp = _agg_case(seed=8)
    pred = E.BloomFilterMightContain(E.Literal(data, T.binary), E.XxHash64(E.Column("k")), "rf")
    partial, final = _agg_plans(rb, pred)
    mid = PL.collect(partial)
    fin_leaf = PL.MemoryExec.from_arrow(mid, mid[0].schema)
    gk = [E.GroupingExpr("g", E.Column("g"))]
    ins = fin_leaf.schema()
    final2 = PL.AggExec(PL.HashAgg, gk, [E.AggExpr("s", E.FINAL, PL.create_agg(E.AGG_SUM, [E.placeholder(T.int64)], ins, T.int64)),
                                         E.AggExpr("c", E.FINAL, PL.create_agg(E.AGG_COUNT, [E.placeholder(T.int64)], ins, T.int64))], False, fin_leaf)
    assert _rows(PL.collect(final2)) == exp


def test_plans_without_bloom_keep_their_fast_kernels():
    rb, _, _ = _agg_case(n=100_000)
    _, final = _agg_plans(rb, E.BinaryExpr(E.Column("k"), "Lt", E.Literal(10_000, T.int64)))
    PL.collect(final)
    assert final.last_metrics["fast_path_launches"] > 0


def test_more_than_four_filters_in_one_program_are_unsupported():
    data = build_filter([1], 64, 1)
    rb = probe_table(100, seed=2, keys=[1])
    preds = [E.BloomFilterMightContain(E.Literal(data, T.binary), E.Column("v"), f"u{i}") for i in range(5)]
    with pytest.raises(native.NativeError) as ei:
        PL.collect(PL.FilterExec(preds, PL.MemoryExec.from_arrow([rb], rb.schema)))
    assert ei.value.code == native.ERR_UNSUPPORTED and "more than 4 BloomFilterMightContain" in ei.value.msg
    PL.collect(PL.FilterExec(preds[:4], PL.MemoryExec.from_arrow([rb], rb.schema)))


# ---- scalar subquery resolved at op create ----------------------------------------------------------------------------
def test_resolver_hands_the_filter_to_might_contain_once_per_op():
    keys = np.random.default_rng(11).integers(0, 10**6, 5_000).tolist()
    hk = [B.xxhash64(int(x).to_bytes(8, "little", signed=True), 42) for x in keys]
    data = build_filter(hk, 1 << 16, 4)
    calls = []

    def resolve(serialized):
        calls.append(serialized)
        return data if serialized == b"subquery#1" else None
    rng = np.random.default_rng(12)
    probe = np.concatenate([np.asarray(keys, np.int64), rng.integers(0, 10**6, 50_000, dtype=np.int64)])
    rb = pa.RecordBatch.from_arrays([pa.array(probe), pa.array(np.arange(len(probe), dtype=np.int64))], names=["k", "row"])
    native.set_scalar_subquery_resolver(resolve)
    try:
        for serialized, nonempty in ((b"subquery#1", True), (b"subquery#null", False)):
            calls.clear()
            pred = E.BloomFilterMightContain(E.ScalarSubquery(serialized), E.XxHash64(E.Column("k")), "rf")
            got = PL.collect(PL.FilterExec([pred], PL.MemoryExec.from_arrow(batches_of(rb, 20_000), rb.schema)))
            assert calls == [serialized]
            rows = sorted(r for b in got for r in b.column(1).to_pylist())
            if nonempty:
                assert set(range(len(keys))) <= set(rows)                 # no inserted key is dropped
                m = B.might_contain(data, B.spark_xxhash64([probe.tolist()], ["int64"]))
                assert rows == [i for i, x in enumerate(m) if x]
            else:
                assert rows == []                                         # a NULL filter keeps no row
    finally:
        native.set_scalar_subquery_resolver(None)


# ---- BLOOM_FILTER aggregate (the creation side) ----------------------------------------------------------------------
EST, NBITS = 5_000, 1 << 16
KS = T.Schema([T.Field("k", T.int64, True), T.Field("f", T.int64, False)])


def _key_batches(seed, n=40_000, parts=4, null_frac=0.1):
    rng = np.random.default_rng(seed)
    k = rng.integers(-2**40, 2**40, n, dtype=np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(k, mask=rng.random(n) < null_frac), pa.array(rng.integers(0, 10, n, dtype=np.int64))], names=["k", "f"])
    return batches_of(rb, (n + parts - 1) // parts)


def _bloom_aggs(mode, child, schema, est=EST, nbits=NBITS, name="bf"):
    return [E.AggExpr(name, mode, PL.create_agg(E.AGG_BLOOM_FILTER, [child, E.Literal(est, T.int64), E.Literal(nbits, T.int64)], schema, T.binary))]


def _partial(batches, with_filter=False, hashed=True):
    leaf = PL.MemoryExec.from_arrow(batches, batches[0].schema) if batches else PL.MemoryExec(KS)
    src = PL.FilterExec([E.BinaryExpr(E.Column("f"), "Lt", E.Literal(5, T.int64))], leaf) if with_filter else leaf
    value = E.XxHash64(E.Column("k")) if hashed else E.Column("k")
    return PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.PARTIAL, value, KS), False, src)


def _expected_filter(batches, with_filter=False):
    """XxHash64 of a NULL key is the seed's hash (never NULL), so every kept row puts a value"""
    vals = []
    for b in batches:
        keep = [k for k, f in zip(col(b, "k"), col(b, "f")) if not with_filter or f < 5]
        vals.append(B.spark_xxhash64([keep], ["int64"]))
    return B.bloom_agg(vals, EST, NBITS)


def _binary_cell(batches, name=E.AGG_BUF_COLUMN_NAME):
    assert sum(b.num_rows for b in batches) == 1
    b = next(b for b in batches if b.num_rows)
    return b.column(b.schema.get_field_index(name))[0].as_py()


@pytest.mark.parametrize("with_filter", [False, True])
def test_bloom_agg_fused_partial_final_bytes(with_filter):
    batches = _key_batches(21, n=150)                                  # few keys: shrink_to_fit folds the filter
    p = _partial(batches, with_filter)
    final = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), p.schema()), False, p)
    got = _binary_cell(PL.collect(final), "bf")
    exp = _expected_filter(batches, with_filter)
    assert got == B.final_bytes(exp)                                   # shrink_to_fit + write_to, byte for byte
    assert len(got) < 12 + 8 * (NBITS // 64)                           # the shrink took place
    assert final.last_metrics["gpu_kernel_launches"] > 0


@pytest.mark.parametrize("columnar", [False, True])
def test_bloom_agg_partial_partial_merge_final_as_ops(columnar):
    conf = native.default_conf(partial_state_columnar=int(columnar))
    parts = [_key_batches(s) for s in (1, 2, 3)]
    name = "bf" if columnar else E.AGG_BUF_COLUMN_NAME
    states = []
    for batches in parts:
        p = _partial(batches)
        out = PL.collect(p, conf)
        exp = _expected_filter(batches)
        assert _binary_cell(out, name) == (exp.write_to() if columnar else B.frozen_row(exp))   # the unshrunk state
        states += out
    sschema = T.from_arrow_schema(states[0].schema)
    union = _expected_filter([b for batches in parts for b in batches])
    merge = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.PARTIAL_MERGE, E.placeholder(T.binary), sschema), False, PL.MemoryExec.from_arrow(states, states[0].schema), columnar_state=columnar)
    merged = PL.collect(merge, conf)
    assert _binary_cell(merged, name) == (union.write_to() if columnar else B.frozen_row(union))
    final = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), sschema), False, PL.MemoryExec.from_arrow(states, states[0].schema))
    assert _binary_cell(PL.collect(final, conf), "bf") == B.final_bytes(union)


def test_bloom_agg_none_cases():
    """no row pushed: the accumulator stays None ([0], then NULL); a batch of only NULL values creates the (empty) filter"""
    p = _partial([])
    out = PL.collect(p)
    assert _binary_cell(out) == b"\x00"
    fin = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), p.schema()), False, PL.MemoryExec.from_arrow(out, out[0].schema))
    assert _binary_cell(PL.collect(fin), "bf") is None
    nulls = pa.RecordBatch.from_arrays([pa.array([None] * 100, pa.int64()), pa.array(np.zeros(100, np.int64))], names=["k", "f"])
    p = _partial([nulls], hashed=False)
    out = PL.collect(p)
    empty = B.bloom_agg([[None] * 100], EST, NBITS)
    assert empty is not None and empty.bits.true_count() == 0 and _binary_cell(out) == B.frozen_row(empty)
    fin = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), p.schema()), False, PL.MemoryExec.from_arrow(out, out[0].schema))
    assert _binary_cell(PL.collect(fin), "bf") == B.final_bytes(empty) == B.SparkBloomFilter(empty.k, B.SparkBitArray([0])).write_to()


def test_bloom_agg_merge_of_different_filters_is_invalid_arg():
    a = PL.collect(_partial(_key_batches(5)))
    other = _key_batches(6)
    p2 = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.PARTIAL, E.XxHash64(E.Column("k")), KS, est=50), False, PL.MemoryExec.from_arrow(other, other[0].schema))
    b = PL.collect(p2)
    fin = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), T.from_arrow_schema(a[0].schema)), False, PL.MemoryExec.from_arrow(a + b, a[0].schema))
    with pytest.raises(native.NativeError) as ei:
        PL.collect(fin)
    assert ei.value.code == native.ERR_INVALID_ARG and "put_all needs equal k and size" in ei.value.msg


def test_bloom_agg_through_shuffle_and_ipc_reader(tmp_path):
    import struct
    parts = [_key_batches(s) for s in (7, 8)]
    blocks = []
    for m, batches in enumerate(parts):
        w = PL.ShuffleWriterExec(_partial(batches), ("single",), str(tmp_path / f"m{m}.data"), str(tmp_path / f"m{m}.index"))
        PL.collect(w)
        data, index = open(w.output_data_file, "rb").read(), open(w.output_index_file, "rb").read()
        offs = struct.unpack("<%dq" % (len(index) // 8), index)
        blocks.append(data[offs[0]:offs[1]])
    pschema = _partial(parts[0]).schema()
    fin = PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), pschema), False, PL.IpcReaderExec(pschema, blocks))
    assert _binary_cell(PL.collect(fin), "bf") == B.final_bytes(_expected_filter([b for batches in parts for b in batches]))


def test_gpu_built_filter_feeds_might_contain_through_the_resolver():
    """the aggregate builds the filter on the GPU; a resolver hands its bytes to a second op's might_contain, once per op"""
    build = _key_batches(31, n=20_000)
    p = _partial(build)
    fbytes = _binary_cell(PL.collect(PL.AggExec(PL.HashAgg, [], _bloom_aggs(E.FINAL, E.placeholder(T.binary), p.schema()), False, p)), "bf")
    calls = []
    native.set_scalar_subquery_resolver(lambda s: calls.append(s) or fbytes)
    try:
        probe = batches_of(pa.Table.from_batches(build).combine_chunks().to_batches()[0], 7_000)
        pred = E.BloomFilterMightContain(E.ScalarSubquery(b"sq"), E.XxHash64(E.Column("k")), "rf")
        got = PL.collect(PL.FilterExec([pred], PL.MemoryExec.from_arrow(probe, probe[0].schema)))
        assert calls == [b"sq"]
        kept = [k for b in got for k in col(b, "k")]
        inserted = [k for b in build for k in col(b, "k") if k is not None]
        assert set(inserted) <= set(kept)                               # no inserted key is dropped
        exp = B.might_contain(fbytes, B.spark_xxhash64([[k for b in probe for k in col(b, "k")]], ["int64"]))
        assert len(kept) == sum(exp)
    finally:
        native.set_scalar_subquery_resolver(None)
