"""Utf8 columns on the GPU path, through the C ABI, against the string oracle (oracle/string_oracle.py): string predicates,
comparisons, IN lists, TryCast(Utf8 -> int), Utf8 columns carried through FilterExec / ProjectExec (host and device input and
output), fused Filter -> Agg over string predicates, and the plans that stay off the device."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from oracle import string_oracle as S
from string_kat_cases import STRING_MATCH_KATS, STRING_TO_BIGINT_KAT, TO_LONG_EDGE_CASES

pytestmark = pytest.mark.gpu

U = T.utf8


def run(rb_or_batches, predicates, projections, conf=None, batch_rows=10000):
    batches = rb_or_batches if isinstance(rb_or_batches, list) else [rb_or_batches.slice(i, batch_rows) for i in range(0, max(rb_or_batches.num_rows, 1), batch_rows)]
    leaf = PL.MemoryExec.from_arrow(batches, batches[0].schema)
    plan = PL.FilterExec(predicates, leaf) if predicates else leaf
    if projections is not None:
        plan = PL.ProjectExec(projections, plan)
    got = PL.collect(plan, conf)
    exp = S.filter_project(predicates, projections, leaf.schema(), batches)
    assert S.rows_of(got) == exp
    return got, plan


def string_table(n, seed=0, null_frac=0.1, long_every=0):
    rng = np.random.default_rng(seed)
    alphabet = np.array(list("abcxyz") + ["é", "€", "\U0001F600", "ab", "xyz"])
    def col():
        out = []
        for i in range(n):
            r = rng.random()
            if r < null_frac:
                out.append(None)
            elif r < null_frac + 0.05:
                out.append("")
            else:
                out.append("".join(rng.choice(alphabet, rng.integers(1, 8))))
            if long_every and i % long_every == long_every - 1:
                out[-1] = "ab" * int(rng.integers(2048, 4096))
        return pa.array(out, pa.string())
    k = pa.array(np.arange(n, dtype=np.int64))
    return pa.RecordBatch.from_arrays([k, col(), col(), col()], names=["k", "s", "t", "u"])


# ---- known answers ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", STRING_MATCH_KATS, ids=[c[0] for c in STRING_MATCH_KATS])
def test_string_match_kats(case):
    _, values, kind, pattern, scalar, expected = case
    rb = pa.RecordBatch.from_arrays([pa.array(values, pa.string())], names=["s"])
    operand = E.Column("s") if scalar is None else E.Literal(scalar, U)
    got, _ = run(rb, [], [(E.StringMatch(kind, operand, pattern), "r")])
    assert [r[0] for r in S.rows_of(got)] == expected


def test_string_to_bigint_kat():
    rb = pa.RecordBatch.from_arrays([pa.array([v for v, _ in STRING_TO_BIGINT_KAT], pa.string())], names=["s"])
    got, _ = run(rb, [], [(E.TryCast(E.Column("s"), T.int64), "r")])
    assert [r[0] for r in S.rows_of(got)] == [e for _, e in STRING_TO_BIGINT_KAT]


def test_to_long_edge_cases_every_width():
    rb = pa.RecordBatch.from_arrays([pa.array([s for s, _, _ in TO_LONG_EDGE_CASES], pa.string())], names=["s"])
    projections = [(E.TryCast(E.Column("s"), t), f"i{t.bit_width}") for t in (T.int8, T.int16, T.int32, T.int64)]
    got, _ = run(rb, [], projections)
    rows = S.rows_of(got)
    for (s, bits, expected), row in zip(TO_LONG_EDGE_CASES, rows):
        assert row[[8, 16, 32, 64].index(bits)] == expected, s


# ---- predicates ------------------------------------------------------------------------------------------------------------
PREDICATES = [
    E.StartsWith(E.Column("s"), "ab"), E.EndsWith(E.Column("s"), "z"), E.Contains(E.Column("s"), "xyz"), E.Contains(E.Column("s"), ""),
    E.StartsWith(E.Column("s"), "é"), E.Contains(E.Column("s"), "\U0001F600a"),
    E.BinaryExpr(E.Column("s"), "Eq", E.Literal("ab", U)), E.BinaryExpr(E.Column("s"), "NotEq", E.Literal("", U)),
    E.BinaryExpr(E.Column("s"), "Lt", E.Literal("b", U)), E.BinaryExpr(E.Column("s"), "LtEq", E.Literal("ab", U)),
    E.BinaryExpr(E.Column("s"), "Gt", E.Literal("é", U)), E.BinaryExpr(E.Literal("c", U), "GtEq", E.Column("s")),
    E.BinaryExpr(E.Column("s"), "Lt", E.Column("t")), E.BinaryExpr(E.Column("s"), "GtEq", E.Column("t")),
    E.BinaryExpr(E.Column("s"), "Eq", E.Column("t")),
    E.InList(E.Column("s"), [E.Literal(x, U) for x in ("a", "ab", "", "é€")]),
    E.InList(E.Column("s"), [E.Literal(x, U) for x in ("a", "b")], negated=True),
    E.InList(E.Column("s"), [E.Literal("a", U), E.Literal(None, U)]),
    E.IsNull(E.Column("s")), E.IsNotNull(E.Column("t")),
    E.BinaryExpr(E.StartsWith(E.Column("s"), "a"), "Or", E.Contains(E.Column("t"), "y")),
    E.BinaryExpr(E.TryCast(E.Column("s"), T.int64), "Gt", E.Literal(0, T.int64)),
    E.InList(E.Column("s"), [E.Literal("ab", U), E.Literal(None, T.null)], negated=True),       # an untyped NULL item arrives as TryCast(NULL)
]


@pytest.mark.parametrize("pi", range(len(PREDICATES)))
def test_every_string_predicate(pi):
    run(string_table(20_000, seed=pi), [PREDICATES[pi]], [(E.Column("k"), "k"), (E.Column("s"), "s"), (E.Column("t"), "t")])


# ---- carrying Utf8 columns -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncols", [1, 2, 3])
@pytest.mark.parametrize("sel", ["none", "half", "all"])
def test_carry_utf8_columns(ncols, sel):
    pred = {"none": E.BinaryExpr(E.Column("k"), "Lt", E.Literal(0, T.int64)),
            "half": E.BinaryExpr(E.Column("k"), "Lt", E.Literal(15_000, T.int64)),
            "all": E.BinaryExpr(E.Column("k"), "GtEq", E.Literal(0, T.int64))}[sel]
    cols = [(E.Column(c), c) for c in ["s", "t", "u"][:ncols]]
    got, _ = run(string_table(30_000, seed=ncols), [pred], [(E.Column("k"), "k")] + cols)
    assert sum(b.num_rows for b in got) == {"none": 0, "half": 15_000, "all": 30_000}[sel]


def test_project_without_filter_and_identity():
    rb = string_table(25_000, seed=3)
    run(rb, [], [(E.Column("t"), "t"), (E.Column("k"), "k"), (E.Column("s"), "s")])
    run(rb, [], None)
    run(rb, [E.BinaryExpr(E.Column("k"), "Lt", E.Literal(7000, T.int64))], None)     # FilterExec only: every column carried


def test_filter_over_an_unreferenced_string_column():
    rb = string_table(20_000, seed=4)
    got, plan = run(rb, [E.BinaryExpr(E.Column("k"), "Lt", E.Literal(1234, T.int64))], [(E.Column("k"), "k")])
    assert sum(b.num_rows for b in got) == 1234


def test_sliced_host_input():
    rb = string_table(40_000, seed=5)
    batches = [rb.slice(3, 17_000), rb.slice(17_003, 5), rb.slice(20_001, 19_000)]
    pred = [E.Contains(E.Column("s"), "a")]
    run(batches, pred, [(E.Column("s"), "s"), (E.Column("k"), "k")])
    run(batches, pred, [(E.Column("s"), "s")], conf=native.default_conf(staging_rows=0))          # direct import path


def test_many_small_pushes_and_staging_growth():
    # 10 k-row pushes go through the staging ring (a push stages when it is shorter than staging_rows / 2); about 1.2 MB of long strings
    # per push exceed the ring's staging_rows x 32 = 800 KB of string bytes and grow its data buffer
    rb = string_table(60_000, seed=6, long_every=50)
    batches = [rb.slice(i, 10_000) for i in range(0, 60_000, 10_000)]
    got, _ = run(batches, [E.StartsWith(E.Column("s"), "ab")], [(E.Column("s"), "s"), (E.Column("t"), "t")],
                 conf=native.default_conf(staging_rows=25_000))
    assert max(len(r[0]) for r in S.rows_of(got)) >= 4096


def test_long_strings_all_null_and_empty():
    big = "x" * (1 << 20)
    vals = ["a" * 4096, big, "", None, "ab" * 5000 + "xyz", "", "x"]
    rb = pa.RecordBatch.from_arrays([pa.array(np.arange(len(vals), dtype=np.int64)), pa.array(vals, pa.string()),
                                     pa.array([None] * len(vals), pa.string())], names=["k", "s", "n"])
    got, _ = run(rb, [E.Contains(E.Column("s"), "xyz")], [(E.Column("s"), "s")])
    assert S.rows_of(got) == [(("ab" * 5000 + "xyz").encode(),)]
    got, _ = run(rb, [E.BinaryExpr(E.Column("k"), "NotEq", E.Literal(0, T.int64))], [(E.Column("s"), "s"), (E.Column("n"), "n")])
    assert S.rows_of(got)[0][0] == big.encode()
    run(rb, [E.IsNull(E.Column("n"))], [(E.Column("n"), "n"), (E.Column("s"), "s")])


def test_output_schema_format_is_u():
    rb = string_table(100, seed=7)
    plan = PL.ProjectExec([(E.Column("s"), "s")], PL.FilterExec([E.IsNotNull(E.Column("s"))], PL.MemoryExec.from_arrow([rb])))
    with native.NativeOp(plan.plan_bytes()) as op:
        assert op.output_schema().field("s").type == pa.string()
        assert op.input_schema().field("t").type == pa.string()


# ---- device input and output -----------------------------------------------------------------------------------------------
def _device_batch(rb, torch):
    cols, keep = [], []
    for c in rb.columns:
        if pa.types.is_string(c.type):
            assert c.offset == 0
            offs = torch.tensor(np.frombuffer(c.buffers()[1], np.int32)[: len(c) + 1].copy(), device="cuda")
            data = torch.tensor(np.frombuffer(c.buffers()[2], np.uint8).copy() if c.buffers()[2] is not None else np.zeros(1, np.uint8), device="cuda")
            valid = torch.tensor(np.frombuffer(c.buffers()[0], np.uint8).copy(), device="cuda") if c.null_count else None
            cols.append((data.data_ptr(), valid.data_ptr() if valid is not None else 0, len(c), offs.data_ptr()))
            keep += [offs, data] + ([valid] if valid is not None else [])
        else:
            v = torch.tensor(c.to_numpy(), device="cuda")
            cols.append((v.data_ptr(), 0, len(c))); keep.append(v)
    return native.DeviceBatch(cols, rb.num_rows, 0, keep)


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
def test_push_device_and_pull_device(null_frac):
    torch = pytest.importorskip("torch")
    rb = string_table(30_000, seed=8, null_frac=null_frac)
    schema = T.from_arrow_schema(rb.schema)
    pred = [E.InList(E.Column("s"), [E.Literal(x, U) for x in ("a", "b", "ab", "xyz")], negated=True)]
    proj = [(E.Column("k"), "k"), (E.Column("s"), "s"), (E.Column("u"), "u")]
    plan = PL.ProjectExec(proj, PL.FilterExec(pred, PL.MemoryExec(schema)))
    exp = S.filter_project(pred, proj, schema, [rb])
    with native.NativeOp(plan.plan_bytes()) as op:
        op.push_device(_device_batch(rb, torch))
        op.finish()
        got = op.pull_all()
    assert S.rows_of(got) == exp
    # pull_device -> push_device_array into an identity projection -> host
    with native.NativeOp(plan.plan_bytes()) as op:
        op.push_device(_device_batch(rb, torch))
        op.finish()
        outs = []
        while (d := op.pull_device()) is not None:
            outs.append(d)
    out_schema = T.Schema([T.Field("k", T.int64, False), T.Field("s", U, True), T.Field("u", U, True)])
    ident = PL.ProjectExec([(E.Column("s"), "s"), (E.Column("k"), "k")], PL.MemoryExec(out_schema))
    with native.NativeOp(ident.plan_bytes()) as op2:
        for d in outs:
            op2.push_device_array(d)
        op2.finish()
        rows = S.rows_of(op2.pull_all())
    assert rows == [(s, k) for k, s, _ in exp]


@pytest.mark.parametrize("offset", [8, 16_000])
def test_direct_import_slice_without_filter(offset):
    # a direct import copies only the referenced string bytes and rebases the offsets; without a filter the column is then carried
    # as it is (ProjectExec and the identity path), so the exported bytes must be the slice's own
    rb = string_table(40_000, seed=14)
    batches = [rb.slice(offset, 20_000), rb.slice(offset + 20_000, 4_000)]
    conf = native.default_conf(staging_rows=0)
    run(batches, [], [(E.Column("k"), "k"), (E.Column("s"), "s")], conf=conf)
    run(batches, [], None, conf=conf)


def test_misaligned_long_strings():
    # 64-400 byte strings land at every alignment of source and destination: the shifted 16-byte copies of the gather
    rng = np.random.default_rng(15)
    vals = ["".join(chr(97 + int(x)) for x in rng.integers(0, 26, int(n))) for n in rng.integers(60, 400, 3000)]
    rb = pa.RecordBatch.from_arrays([pa.array(np.arange(len(vals), dtype=np.int64)), pa.array(vals, pa.string())], names=["k", "s"])
    for pred in (E.BinaryExpr(E.Column("k"), "NotEq", E.Literal(0, T.int64)), E.Contains(E.Column("s"), "q")):
        run(rb, [pred], [(E.Column("s"), "s"), (E.Column("k"), "k")])


def _sliced(rb, torch, offset, length):
    db = _device_batch(rb, torch)
    for i in range(db.n):
        db.children[i].offset = offset
    db.dev.array.length = length
    return db


@pytest.mark.parametrize("with_filter", [False, True])
def test_sliced_device_input(with_filter):
    torch = pytest.importorskip("torch")
    rb = string_table(5_000, seed=9, null_frac=0.0)
    schema = T.from_arrow_schema(rb.schema)
    pred = [E.StartsWith(E.Column("t"), "a")] if with_filter else []
    proj = [(E.Column("s"), "s"), (E.Column("t"), "t")]
    plan = PL.ProjectExec(proj, PL.FilterExec(pred, PL.MemoryExec(schema)) if pred else PL.MemoryExec(schema))
    with native.NativeOp(plan.plan_bytes()) as op:
        op.push_device(_sliced(rb, torch, 123, 4_000))
        op.finish()
        assert S.rows_of(op.pull_all()) == S.filter_project(pred, proj, schema, [rb.slice(123, 4_000)])


# ---- literal pool ------------------------------------------------------------------------------------------------------------
def test_literal_pool_bound():
    rb = string_table(1_000, seed=10)
    items = [chr(65 + i) * 256 for i in range(16)]                                   # exactly 4096 bytes
    run(rb, [E.InList(E.Column("s"), [E.Literal(x, U) for x in items])], [(E.Column("k"), "k")])
    over = PL.FilterExec([E.InList(E.Column("s"), [E.Literal(x, U) for x in items + ["z"]])], PL.MemoryExec.from_arrow([rb]))
    with pytest.raises(native.NativeError) as ei:
        PL.collect(over)
    assert ei.value.code == native.ERR_UNSUPPORTED and "literal pool" in ei.value.msg


# ---- aggregates ----------------------------------------------------------------------------------------------------------
def _agg_plan(rb, pred, aggs_of):
    leaf = PL.MemoryExec.from_arrow([rb.slice(i, 10_000) for i in range(0, rb.num_rows, 10_000)])
    ins = leaf.schema()
    g = [E.GroupingExpr("g", E.Column("g"))]
    partial = PL.AggExec(PL.HashAgg, g, aggs_of(E.PARTIAL, ins), False, PL.FilterExec(pred, leaf) if pred else leaf)
    return PL.AggExec(PL.HashAgg, g, aggs_of(E.FINAL, ins), False, partial)


def numeric_strings(n, seed):
    rng = np.random.default_rng(seed)
    vals = [str(int(v)) for v in rng.integers(-10**12, 10**12, n)]
    for i in rng.choice(n, n // 100, replace=False):
        vals[i] = ["x1", "", "1.5", "-", "12a", None][int(i) % 6]
    return vals


@pytest.mark.parametrize("generic", [0, 1])
def test_fused_filter_agg_with_string_predicate(generic):
    n = 50_000
    rng = np.random.default_rng(11)
    ns = numeric_strings(n, 11)
    rb = pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 100, n)), pa.array(ns, pa.string()), pa.array(rng.integers(0, 1000, n))],
                                    names=["g", "ns", "v"])
    pred = [E.BinaryExpr(E.StartsWith(E.Column("ns"), "1"), "Or", E.Contains(E.Column("ns"), "99"))]

    def aggs(mode, ins):
        ph = mode == E.FINAL
        return [E.AggExpr("sv", mode, PL.create_agg(E.AGG_SUM, [E.placeholder(T.int64) if ph else E.Column("v")], ins, T.int64)),
                E.AggExpr("sn", mode, PL.create_agg(E.AGG_SUM, [E.placeholder(T.int64) if ph else E.TryCast(E.Column("ns"), T.int64)], ins, T.int64)),
                E.AggExpr("cn", mode, PL.create_agg(E.AGG_COUNT, [E.placeholder(T.int64) if ph else E.Column("ns")], ins, T.int64))]
    got = PL.collect(_agg_plan(rb, pred, aggs), native.default_conf(force_generic_kernels=generic))
    exp = {}
    for g, s, v in zip(rb.column("g").to_pylist(), ns, rb.column("v").to_pylist()):
        if s is None or not (s.startswith("1") or "99" in s):
            continue
        e = exp.setdefault(g, [0, None, 0])
        e[0] += v
        x = S.to_long(s.encode())
        if x is not None:
            e[1] = (e[1] or 0) + x
        e[2] += 1
    rows = {r[0]: list(r[1:]) for r in S.rows_of(got)}
    assert rows == exp


def test_count_and_sum_of_trycast_over_strings():
    n = 30_000
    rng = np.random.default_rng(12)
    ns = numeric_strings(n, 12)
    rb = pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 50, n)), pa.array(ns, pa.string())], names=["g", "ns"])

    def aggs(mode, ins):
        ph = mode == E.FINAL
        return [E.AggExpr("c", mode, PL.create_agg(E.AGG_COUNT, [E.placeholder(T.int64) if ph else E.Column("ns")], ins, T.int64)),
                E.AggExpr("s", mode, PL.create_agg(E.AGG_SUM, [E.placeholder(T.int64) if ph else E.TryCast(E.Column("ns"), T.int64)], ins, T.int64))]
    rows = {r[0]: list(r[1:]) for r in S.rows_of(PL.collect(_agg_plan(rb, [], aggs)))}
    exp = {}
    for g, s in zip(rb.column("g").to_pylist(), ns):
        e = exp.setdefault(g, [0, None])
        if s is not None:
            e[0] += 1
            x = S.to_long(s.encode())
            if x is not None:
                e[1] = (e[1] or 0) + x
    assert rows == exp


# ---- what stays off the device ----------------------------------------------------------------------------------------------
def _unsupported(make):
    with pytest.raises(native.NativeError) as ei:
        PL.collect(make())
    assert ei.value.code == native.ERR_UNSUPPORTED, ei.value.msg
    return ei.value.msg


def test_unsupported_plans(tmp_path):
    rb = string_table(100, seed=13)
    leaf = lambda: PL.MemoryExec.from_arrow([rb])
    ins = leaf().schema()
    assert "utf8" in _unsupported(lambda: PL.ProjectExec([(E.Literal("x", U), "x")], leaf()))
    assert "utf8" in _unsupported(lambda: PL.ProjectExec([(E.Case(None, [(E.IsNull(E.Column("s")), E.Literal("a", U))], E.Literal("b", U)), "c")], leaf()))
    assert "CASE" in _unsupported(lambda: PL.FilterExec([E.BinaryExpr(E.Case(None, [(E.IsNull(E.Column("s")), E.Literal("a", U))], E.Column("t")), "Eq", E.Literal("a", U))], leaf()))
    assert "NullIf" in _unsupported(lambda: PL.FilterExec([E.IsNull(E.ScalarFunction("NullIf", [E.Column("s"), E.Literal("", U)], U))], leaf()))
    assert "NullIf" in _unsupported(lambda: PL.FilterExec([E.BinaryExpr(E.ScalarFunction("NullIf", [E.Column("s"), E.Literal("TN", U)], U), "Eq", E.Literal("TN", U))], leaf()))
    assert "NullIfZero" in _unsupported(lambda: PL.FilterExec([E.IsNull(E.ScalarFunction("NullIfZero", [E.Column("s")], U))], leaf()))
    # 32 fixed-width outputs plus the selection vector of a carried string column: one output over the device limit
    wide = pa.RecordBatch.from_arrays([pa.array(np.arange(10, dtype=np.int64)) for _ in range(32)] + [pa.array(["x"] * 10, pa.string())],
                                      names=[f"c{i}" for i in range(32)] + ["s"])
    assert "outputs" in _unsupported(lambda: PL.FilterExec([E.BinaryExpr(E.Column("c0"), "Lt", E.Literal(5, T.int64))], PL.MemoryExec.from_arrow([wide])))
    _unsupported(lambda: PL.ProjectExec([(E.ScalarFunction("Substring", [E.Column("s")], U), "x")], leaf()))
    _unsupported(lambda: PL.ProjectExec([(E.TryCast(E.Column("k"), U), "x")], leaf()))
    assert "cast" in _unsupported(lambda: PL.ProjectExec([(E.Cast(E.Column("s"), T.int64), "x")], leaf()))
    assert "grouping" in _unsupported(lambda: PL.AggExec(PL.HashAgg, [E.GroupingExpr("s", E.Column("s"))],
                                                         [E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Column("k")], ins, T.int64))], False, leaf()))
    for fn in (E.AGG_MIN, E.AGG_MAX):
        _unsupported(lambda: PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], [E.AggExpr("m", E.PARTIAL, PL.create_agg(fn, [E.Column("s")], ins, U))], False, leaf()))
    for fn in (E.AGG_SUM, E.AGG_AVG):
        assert "utf8" in _unsupported(lambda: PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))],
                                                         [E.AggExpr("m", E.PARTIAL, PL.create_agg(fn, [E.Column("s")], ins, T.int64 if fn == E.AGG_SUM else T.float64))], False, leaf()))
    assert "SortExec" in _unsupported(lambda: PL.SortExec(leaf(), [(E.Column("k"), False, True)]))
    assert "shuffle" in _unsupported(lambda: PL.ShuffleWriterExec(leaf(), ("hash", [E.Column("k")], 4), str(tmp_path / "d"), str(tmp_path / "i")))
    assert "join" in _unsupported(lambda: PL.BroadcastJoinBuildHashMapExec(leaf(), [E.Column("k")]))
    pq = tmp_path / "s.parquet"
    import pyarrow.parquet as papq
    papq.write_table(pa.Table.from_batches([rb]), pq)
    assert "ParquetScanExec" in _unsupported(lambda: PL.ParquetScanExec(ins, [(str(pq), 0, None)], projection=[0, 1]))
