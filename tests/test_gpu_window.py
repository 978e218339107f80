"""WindowExec on the GPU against the oracle (oracle/window_oracle.py): the reference's KATs, every function over every fixed-width
key type, batch splits inside and on partition boundaries, host and device input / output, aggregate edges, the group limit
(WindowGroupLimit) with the combining rule, whole ops (Sort -> Window, Filter/Project -> Window -> Filter), and the refusals."""
import decimal
import zlib

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from oracle import blaze_oracle as O
from oracle import window_oracle as W
import exact_agg as X
from helpers import with_nulls, split_batches
from window_cases import KATS, brute_force, gpu_plan, kat_input, kat_window, oracle_run, sorted_table, window_expr

pytestmark = pytest.mark.gpu
UNSTAGED = dict(staging_rows=0)              # every pushed batch reaches the window stage as it is


def conf(**kw):
    return native.default_conf(**kw)


def assert_equal_ordered(gpu_batches, schema, oracle_out, approx_cols=()):
    """window output keeps the input order: values + validity column by column; columns in approx_cols (f64 running sums /
    averages, whose association differs from the row-by-row oracle) within 1e-9 relative, all others bit-exactly"""
    got = O.concat_batches(schema, [O.batch_from_arrow(b) for b in gpu_batches])
    exp = O.concat_batches(schema, oracle_out)
    assert got.num_rows == exp.num_rows, f"row count {got.num_rows} != {exp.num_rows}"
    for i, (g, e) in enumerate(zip(got.cols, exp.cols)):
        assert g.dtype == e.dtype, f"col {i}: dtype {g.dtype} != {e.dtype}"
        assert np.array_equal(g.valid, e.valid), f"col {i} ({schema[i].name}): validity differs"
        gv, ev = g.values[g.valid], e.values[e.valid]
        if schema[i].name in approx_cols:
            np.testing.assert_allclose(gv.astype(np.float64), ev.astype(np.float64), rtol=1e-9, atol=1e-9, err_msg=f"col {schema[i].name}")
        elif g.dtype.is_float:
            w = np.int64 if g.dtype.id == T.FLOAT64 else np.int32
            assert np.array_equal(gv.view(w), ev.view(w)), f"col {i} ({schema[i].name}): float bits differ"
        else:
            assert np.array_equal(gv, ev), f"col {i} ({schema[i].name}): values differ at {np.nonzero(gv != ev)[0][:5]}"


def run_both(schema, batches, exprs, partition, order, group_limit=None, owc=True, cf=None, approx=()):
    plan = gpu_plan(schema, exprs, partition, order, group_limit, owc, batches)
    got = PL.collect(plan, cf or conf(**UNSTAGED))
    osch, exp = oracle_run(schema, exprs, partition, order, batches, group_limit, owc)
    assert_equal_ordered(got, osch, exp, approx)
    return got


# ---- the reference's KATs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch_rows", [None, 1])
@pytest.mark.parametrize("case", KATS, ids=[c["name"] for c in KATS])
def test_kats(case, batch_rows):
    schema, rb = kat_input(case)
    exprs, part, order = kat_window(case, schema)
    batches = [rb] if batch_rows is None else split_batches(rb, batch_rows)
    got = PL.collect(gpu_plan(schema, exprs, part, order, case["group_limit"], case["output_window_cols"], batches), conf(**UNSTAGED))
    t = pa.Table.from_batches(got)
    for name, vals in case["expected"].items():
        assert t.column(name).to_pylist() == vals, name


# ---- random tables vs the oracle: every function, every fixed-width key type ----------------------------------------------------
KEY_TYPES = {
    "int8": (lambda rng, n: rng.integers(-3, 3, n).astype(np.int8), pa.int8()),
    "int16": (lambda rng, n: rng.integers(-3, 3, n).astype(np.int16), pa.int16()),
    "int32": (lambda rng, n: rng.integers(-3, 3, n).astype(np.int32), pa.int32()),
    "int64": (lambda rng, n: rng.integers(-3, 3, n).astype(np.int64) * (1 << 40), pa.int64()),
    "float32": (lambda rng, n: rng.choice(np.array([0.0, -0.0, 1.5, np.nan, -np.inf], np.float32), n), pa.float32()),
    "float64": (lambda rng, n: rng.choice(np.array([0.0, -0.0, 2.25, np.nan, 1e300], np.float64), n), pa.float64()),
    "decimal": (lambda rng, n: [decimal.Decimal(int(x) * 10**20).scaleb(-2) for x in rng.integers(-3, 3, n)], pa.decimal128(30, 2)),
    "bool": (lambda rng, n: rng.integers(0, 2, n).astype(bool), pa.bool_()),
    "date": (lambda rng, n: rng.integers(0, 4, n).astype(np.int32), pa.date32()),
    "timestamp": (lambda rng, n: rng.integers(0, 4, n).astype(np.int64) * 10**6, pa.timestamp("us")),
}


def random_table(key_type, n, seed, null_frac=0.15):
    rng = np.random.default_rng(seed)
    gen, pt = KEY_TYPES[key_type]
    arrs = [with_nulls(rng, np.asarray(gen(rng, n), dtype=object) if key_type == "decimal" else gen(rng, n), null_frac, pt) for _ in range(4)]
    v = with_nulls(rng, rng.integers(-1000, 1000, n).astype(np.int64), 0.2)
    f = with_nulls(rng, rng.integers(-10**6, 10**6, n).astype(np.float64) / 64.0, 0.2)
    rb = pa.RecordBatch.from_arrays(arrs + [v, f], names=["p1", "p2", "o1", "o2", "v", "f"])
    return sorted_table(rb, ["p1", "p2", "o1", "o2"])


ALL_FNS = [("rn", "row_number", None), ("rk", "rank", None), ("dr", "dense_rank", None), ("s", "sum", "v"), ("c", "count", "v"),
           ("mn", "min", "v"), ("mx", "max", "v"), ("a", "avg", "v")]


@pytest.mark.parametrize("key_type", list(KEY_TYPES))
@pytest.mark.parametrize("spec", ["p1|o1", "p1,p2|o1,o2", "|o1", "p1|", "|"])
def test_random_vs_oracle(key_type, spec):
    rb = random_table(key_type, 3_000, seed=zlib.crc32(f"{key_type}{spec}".encode()) % 1000)
    schema = T.from_arrow_schema(rb.schema)
    pnames, onames = [s.split(",") if s else [] for s in spec.split("|")]
    exprs = [window_expr(nm, fn, arg, schema) for nm, fn, arg in ALL_FNS]
    run_both(schema, split_batches(rb, 700), exprs, [E.Column(c) for c in pnames], [(E.Column(c), False, True) for c in onames], approx=("a",))


def test_float_aggregates_and_f64_sums_bit_identical():
    rb = random_table("int32", 20_000, seed=5)
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr("s", "sum", "f", schema), window_expr("a", "avg", "f", schema), window_expr("mn", "min", "f", schema), window_expr("mx", "max", "f", schema)]
    batches = split_batches(rb, 4_096)
    g1 = run_both(schema, batches, exprs, [E.Column("p1")], [(E.Column("o1"), False, True)], approx=("s", "a"))
    g2 = PL.collect(gpu_plan(schema, exprs, [E.Column("p1")], [(E.Column("o1"), False, True)], batches=batches), conf(**UNSTAGED))
    for a, b in zip(g1, g2):
        for name in ("s", "a"):
            assert a.column(name).equals(b.column(name))


# ---- batch splits -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch_rows", [1, 7, 1000, 2048, 5000])
def test_batch_splits(batch_rows):
    rng = np.random.default_rng(batch_rows)
    n = 12_000
    p = np.repeat(np.arange(6), n // 6).astype(np.int64)                     # partitions span many pushes
    o = np.sort(rng.integers(0, 50, n)).astype(np.int64)
    rb = sorted_table(pa.RecordBatch.from_arrays([pa.array(p), pa.array(o), with_nulls(rng, rng.integers(-99, 99, n).astype(np.int64), 0.1)], names=["p", "o", "v"]), ["p", "o"])
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr(nm, fn, arg, schema) for nm, fn, arg in ALL_FNS]
    batches = split_batches(rb, batch_rows) if batch_rows > 1 else split_batches(rb.slice(0, 3000), 1)
    run_both(schema, batches, exprs, [E.Column("p")], [(E.Column("o"), False, True)], approx=("a",))


# ---- input and output paths ---------------------------------------------------------------------------------------------------
def test_host_batches_staged():
    rb = random_table("int64", 50_000, seed=9)
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr(nm, fn, arg, schema) for nm, fn, arg in ALL_FNS]
    run_both(schema, split_batches(rb, 10_000), exprs, [E.Column("p1")], [(E.Column("o1"), False, True)], cf=conf(), approx=("a",))


def test_push_device_and_pull_device():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device for torch")
    n = 40_000
    rng = np.random.default_rng(4)
    p = np.sort(rng.integers(0, 300, n)).astype(np.int64)
    o = rng.integers(0, 5, n).astype(np.int64)
    idx = np.lexsort((o, p)); p, o = p[idx], o[idx]
    v = rng.integers(-10**6, 10**6, n).astype(np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(p), pa.array(o), pa.array(v)], names=["p", "o", "v"])
    schema = T.Schema([T.Field("p", T.int64, False), T.Field("o", T.int64, False), T.Field("v", T.int64, False)])
    exprs = [window_expr("rk", "rank", None, schema), window_expr("s", "sum", "v", schema), window_expr("c", "count", "v", schema)]
    plan = gpu_plan(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)])
    tp, to, tv = (torch.tensor(x, device="cuda") for x in (p, o, v))
    with native.NativeOp(plan.plan_bytes()) as op:
        half = n // 2
        for a, b in ((0, half), (half, n)):
            op.push_device(native.DeviceBatch([(t[a:b].data_ptr(), 0, b - a) for t in (tp, to, tv)], b - a, 0, keepalive=(tp, to, tv)))
        op.finish()
        outs = []
        while (d := op.pull_device()) is not None:
            outs.append(d)
        assert op.metrics()["hot_kernel_rows"] == n            # the copy of the borrowed input columns is not the window stage's hot kernel time
    # the device output pushed into an identity projection, pulled to the host
    out_schema = plan.schema()
    ident = PL.ProjectExec([(E.Column(f.name), f.name) for f in out_schema], PL.MemoryExec(out_schema))
    with native.NativeOp(ident.plan_bytes()) as op2:
        for d in outs:
            op2.push_device_array(d)
        op2.finish()
        got = op2.pull_all()
    osch, exp = oracle_run(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)], [rb])
    assert_equal_ordered(got, osch, exp)


# ---- aggregate edges ----------------------------------------------------------------------------------------------------------
def test_integer_sums_wrap_and_null_prefixes():
    n = 5_000
    rng = np.random.default_rng(2)
    p = np.repeat(np.arange(5), n // 5).astype(np.int64)
    big = rng.integers(1 << 61, 1 << 62, n).astype(np.int64)
    v = with_nulls(rng, big, 0.0)
    mask = np.zeros(n, bool); mask[:300] = True; mask[1000:1100] = True       # NULL prefixes of partitions 0 and 1
    v = pa.array(big, mask=mask)
    i32 = pa.array((big % 2**31).astype(np.int32), mask=mask)
    d = pa.array([decimal.Decimal(int(x) * 10**18) for x in big], pa.decimal128(38, 0), mask=mask)
    rb = pa.RecordBatch.from_arrays([pa.array(p), pa.array(np.arange(n, dtype=np.int64)), v, i32, d], names=["p", "o", "v", "i", "d"])
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr("s64", "sum", "v", schema), window_expr("s32", "sum", "i", schema, T.int32), window_expr("sd", "sum", "d", schema),
             window_expr("ad", "avg", "d", schema, T.decimal128(38, 4)), window_expr("ai", "avg", "i", schema), window_expr("mn", "min", "d", schema),
             window_expr("mx", "max", "v", schema), window_expr("c", "count", "v", schema)]
    run_both(schema, split_batches(rb, 1_500), exprs, [E.Column("p")], [(E.Column("o"), False, True)], approx=("ai",))


# ---- group limit ----------------------------------------------------------------------------------------------------------------
def _limit_table(n=20_000, seed=6):
    """sorted (p, o) with a row id; Utf8 / Binary columns carried through the limit"""
    rng = np.random.default_rng(seed)
    p = np.sort(rng.integers(0, 200, n)).astype(np.int64)
    o = rng.integers(0, 40, n).astype(np.int64)
    idx = np.lexsort((o, p))
    s = pa.array([f"s{x}" if x % 7 else None for x in rng.integers(0, 1000, n)], pa.string())
    b = pa.array([bytes([x % 256]) * (x % 5) for x in rng.integers(0, 1000, n)], pa.binary())
    rb = pa.RecordBatch.from_arrays([pa.array(p[idx]), pa.array(o[idx]), pa.array(np.arange(n, dtype=np.int64)), s, b], names=["p", "o", "rid", "s", "b"])
    return rb, T.from_arrow_schema(rb.schema)


def run_limit(rb, schema, gpu, oracle_exec):
    """`gpu`: a plan over rb's columns; `oracle_exec`: the oracle over the fixed-width columns (p, o, rid).  The carried Utf8 / Binary
    columns must be the input's at each surviving row id."""
    got = PL.collect(gpu, conf(**UNSTAGED))
    fixed = rb.select(["p", "o", "rid"])
    osch, exp = oracle_exec(T.from_arrow_schema(fixed.schema), split_batches(fixed, 3_000))
    t = pa.Table.from_batches(got, schema=T.to_arrow_schema(gpu.schema())) if got else None
    keep = [f.name for f in gpu.schema() if f.name not in ("s", "b")]
    sub = [pa.RecordBatch.from_arrays([b.column(b.schema.get_field_index(c)) for c in keep], names=keep) for b in got]
    assert_equal_ordered(sub, osch, exp)
    if t is not None:
        rid = t.column("rid").combine_chunks()
        assert t.column("s").to_pylist() == rb.column(3).take(rid).to_pylist()
        assert t.column("b").to_pylist() == rb.column(4).take(rid).to_pylist()


@pytest.mark.parametrize("owc", [False, True])
@pytest.mark.parametrize("fn", ["row_number", "rank", "dense_rank"])
@pytest.mark.parametrize("k", [0, 1, 2, 100, 2**31, 2**32 - 1])
def test_group_limit(k, fn, owc):
    rb, schema = _limit_table()
    part, order = [E.Column("p")], [(E.Column("o"), False, True)]
    gpu = gpu_plan(schema, [window_expr("w", fn, None, schema)], part, order, k, owc, split_batches(rb, 3_000))
    run_limit(rb, schema, gpu, lambda fs, bs: oracle_run(fs, [window_expr("w", fn, None, fs)], part, order, bs, k, owc))


def test_window_over_group_limit_combines():
    rb, schema = _limit_table()
    part, order = [E.Column("p")], [(E.Column("o"), False, True)]
    child = PL.WindowExec(PL.MemoryExec(schema, split_batches(rb, 3_000)), [window_expr("w", "rank", None, schema)], part, order, 3, False)
    parent = PL.WindowExec(child, [window_expr("rk", "row_number", None, schema)], part, order)

    def oracle(fs, bs):
        oc = W.WindowExec([window_expr("w", "rank", None, fs)], part, order, fs, 3, False)
        comb = W.WindowExec.combine(W.WindowExec([window_expr("rk", "row_number", None, fs)], part, order, oc.schema), oc)
        return comb.schema, comb.execute([O.batch_from_arrow(b) for b in bs])
    run_limit(rb, schema, parent, oracle)


# ---- whole ops ----------------------------------------------------------------------------------------------------------------
def test_sort_then_window_is_one_op():
    rng = np.random.default_rng(11)
    n = 30_000
    rb = pa.RecordBatch.from_arrays([pa.array(rng.integers(0, 500, n).astype(np.int64)), pa.array(rng.integers(0, 20, n).astype(np.int64)),
                                     pa.array(rng.integers(-50, 50, n).astype(np.int64))], names=["p", "o", "v"])
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr("rk", "rank", None, schema)]
    part, order = [E.Column("p")], [(E.Column("o"), False, True)]
    plan = PL.WindowExec(PL.SortExec(PL.MemoryExec(schema, split_batches(rb, 7_000)), [(E.Column("p"), False, True), (E.Column("o"), False, True)]),
                         exprs, part, order, 5)
    got = PL.collect(plan)
    osch, exp = oracle_run(schema, exprs, part, order, [sorted_table(rb, ["p", "o"])], 5)
    # rows equal in (p, o) may come out of the sort in any order: compare the multisets of rows
    assert O.rows_multiset([O.batch_from_arrow(b) for b in got]) == O.rows_multiset(exp)


def test_filter_project_window_filter_one_op():
    rng = np.random.default_rng(12)
    n = 20_000
    p = np.sort(rng.integers(0, 100, n)).astype(np.int64)
    v = rng.integers(-100, 100, n).astype(np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(p), pa.array(v)], names=["p", "v"])
    schema = T.from_arrow_schema(rb.schema)
    flt = PL.FilterExec([E.BinaryExpr(E.Column("v"), "Gt", E.Literal(-80, T.int64))], PL.MemoryExec(schema, split_batches(rb, 4_000)))
    prj = PL.ProjectExec([(E.Column("p"), "p"), (E.BinaryExpr(E.Column("v"), "Multiply", E.Literal(3, T.int64)), "v3")], flt)
    ps = prj.schema()
    exprs = [window_expr("rk", "row_number", None, ps), E.WindowExpr.agg("s", E.AGG_SUM, [E.BinaryExpr(E.Column("v3"), "Plus", E.Literal(1, T.int64))], T.int64)]
    win = PL.WindowExec(prj, exprs, [E.BinaryExpr(E.Column("p"), "Modulo", E.Literal(50, T.int64))], [])
    top = PL.FilterExec([E.BinaryExpr(E.Column("rk"), "LtEq", E.Literal(10, T.int32))], win)
    with native.NativeOp(top.plan_bytes(), conf(**UNSTAGED)) as op:
        for b in split_batches(rb, 4_000):
            op.push(b)
        op.finish()
        got = op.pull_all()
    ob = O.FilterExec([E.BinaryExpr(E.Column("v"), "Gt", E.Literal(-80, T.int64))], schema).execute([O.batch_from_arrow(b) for b in split_batches(rb, 4_000)])
    ob = O.ProjectExec([(E.Column("p"), "p"), (E.BinaryExpr(E.Column("v"), "Multiply", E.Literal(3, T.int64)), "v3")], schema).execute(ob)
    w = W.WindowExec(exprs, [E.BinaryExpr(E.Column("p"), "Modulo", E.Literal(50, T.int64))], [], ps)
    exp = O.FilterExec([E.BinaryExpr(E.Column("rk"), "LtEq", E.Literal(10, T.int32))], w.schema).execute(w.execute(ob))
    assert_equal_ordered(got, w.schema, exp)


# ---- brute force on the device output -----------------------------------------------------------------------------------------
def test_device_matches_brute_force():
    rb = random_table("float64", 2_000, seed=21)
    schema = T.from_arrow_schema(rb.schema)
    got = pa.Table.from_batches(PL.collect(gpu_plan(schema, [window_expr(nm, fn, arg, schema) for nm, fn, arg in ALL_FNS[:6]],
                                                    [E.Column("p1")], [(E.Column("o1"), False, True)], batches=split_batches(rb, 333)), conf(**UNSTAGED)))
    for nm, fn, arg in ALL_FNS[:6]:
        assert got.column(nm).to_pylist() == brute_force(rb, fn, ["p1"], ["o1"], arg), nm


# ---- numeric edges against the exact reference (tests/exact_agg.py) -------------------------------------------------------------
def _edge_table(groups, dtype):
    """one partition per group, its values in order; o = row number, so every row is its own peer group"""
    p, vals = [], []
    for g, (_kind, v) in enumerate(groups):
        p += [g] * len(v)
        vals += v
    arr = pa.array([None if x is None else x for x in vals], type=dtype)
    rb = pa.RecordBatch.from_arrays([pa.array(np.array(p, np.int64)), pa.array(np.arange(len(p), dtype=np.int64)), arr], names=["p", "o", "x"])
    return rb, T.from_arrow_schema(rb.schema)


def _running_expected(groups, fn, arg_type, result_type):
    out = []
    for _kind, v in groups:
        for i in range(len(v)):
            out.append(X.aggregate(fn, arg_type, result_type, v[: i + 1]))
    return out


def _check_running(got_col, expected, what, may_overflow=None):
    """X.matches row by row.  may_overflow[i]: the running sum's exact value lies beyond DBL_MAX, so it may have rounded to the
    infinity of its sign (the exact reference only calls a sum infinite in every order from 2 * DBL_MAX on, which a prefix of an
    overflowing group can miss); the SUM and the AVG of that row may then be that infinity"""
    def ok(i, e, g):
        if may_overflow and may_overflow[i] and g is not None and np.isinf(g):
            return True
        return X.matches(e, g)
    bad = [(i, e, g) for i, (e, g) in enumerate(zip(expected, got_col)) if not ok(i, e, g)]
    assert not bad, f"{what}: {len(bad)} rows outside the exact reference, first {bad[:3]}"


def test_f64_running_sum_and_avg_within_the_exact_bound():
    groups = X.f64_sum_groups(np.random.default_rng(31), ngroups=140)
    rb, schema = _edge_table(groups, pa.float64())
    exprs = [window_expr("s", "sum", "x", schema), window_expr("a", "avg", "x", schema)]
    got = pa.Table.from_batches(PL.collect(gpu_plan(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)], batches=split_batches(rb, 1_000)), conf(**UNSTAGED)))
    sums = _running_expected(groups, E.AGG_SUM, T.float64, T.float64)
    over = [isinstance(e, X.Interval) and abs(e.center) > X.DBL_MAX for e in sums]
    _check_running(got.column("s").to_pylist(), sums, "SUM", over)
    _check_running(got.column("a").to_pylist(), _running_expected(groups, E.AGG_AVG, T.float64, T.float64), "AVG", over)


def test_f64_running_sum_is_bit_identical_where_the_order_matters():
    """non-dyadic values of mixed magnitude in long partitions that span many tiles and pushes: the rounded sums depend on the
    association, which the tile structure fixes"""
    rng = np.random.default_rng(32)
    n = 200_000
    x = rng.normal(0, 1e6, n) * np.where(rng.random(n) < 0.01, 1e10, 1.0)
    p = np.repeat(np.arange(4), n // 4).astype(np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(p), pa.array(np.arange(n, dtype=np.int64)), pa.array(x)], names=["p", "o", "x"])
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr("s", "sum", "x", schema)]
    runs = [np.concatenate([b.column(3).to_numpy() for b in PL.collect(gpu_plan(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)],
                                                                              batches=split_batches(rb, 50_000)), conf(**UNSTAGED))]) for _ in range(2)]
    assert np.array_equal(runs[0].view(np.int64), runs[1].view(np.int64))
    seq = np.concatenate([np.cumsum(x[p == k]) for k in range(4)])               # one left-to-right association
    assert not np.array_equal(seq.view(np.int64), runs[0].view(np.int64)), "the data must be order-sensitive for this test to mean anything"
    from fractions import Fraction
    for k in range(4):                                                            # every prefix within gamma(m-1) * sum|x| of the exact sum
        xs, got = x[p == k], runs[0][p == k]
        exact, mag = Fraction(0), Fraction(0)
        for m in range(len(xs)):
            exact += Fraction(float(xs[m])); mag += Fraction(abs(float(xs[m])))
            if m % 997 == 0 or m == len(xs) - 1:
                assert abs(Fraction(float(got[m])) - exact) <= X.gamma(m) * mag, (k, m)


@pytest.mark.parametrize("width", [32, 64])
def test_float_running_min_max_edges(width):
    groups = X.float_minmax_groups(np.random.default_rng(33 + width), width, ngroups=220)
    dt = T.float32 if width == 32 else T.float64
    rb, schema = _edge_table(groups, pa.float32() if width == 32 else pa.float64())
    exprs = [window_expr("mn", "min", "x", schema), window_expr("mx", "max", "x", schema)]
    got = pa.Table.from_batches(PL.collect(gpu_plan(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)], batches=split_batches(rb, 500)), conf(**UNSTAGED)))
    for name, fn in (("mn", E.AGG_MIN), ("mx", E.AGG_MAX)):
        col = got.column(name).combine_chunks()
        vals = [None if not ok else (np.float32(v) if width == 32 else float(v)) for ok, v in zip(col.is_valid().to_pylist(), col.fill_null(0).to_numpy())]
        _check_running(vals, _running_expected(groups, fn, dt, dt), name)


@pytest.mark.parametrize("arg_type", [pa.int8(), pa.int16(), pa.int32(), pa.date32(), pa.timestamp("us")])
def test_integer_running_min_max(arg_type):
    rng = np.random.default_rng(34)
    n = 6_000
    np_type = {pa.int8(): np.int8, pa.int16(): np.int16, pa.int32(): np.int32, pa.date32(): np.int32}.get(arg_type, np.int64)
    x = with_nulls(rng, rng.integers(-120, 120, n).astype(np_type), 0.2, arg_type)
    rb = pa.RecordBatch.from_arrays([pa.array(np.repeat(np.arange(30), n // 30).astype(np.int64)), pa.array(np.arange(n, dtype=np.int64)), x], names=["p", "o", "x"])
    schema = T.from_arrow_schema(rb.schema)
    run_both(schema, split_batches(rb, 1_000), [window_expr("mn", "min", "x", schema), window_expr("mx", "max", "x", schema)], [E.Column("p")], [(E.Column("o"), False, True)])


# ---- stage structure ----------------------------------------------------------------------------------------------------------
def test_column_arguments_need_no_projection_stage():
    """SUM over an int64 column carries create_agg's TryCast(v AS int64): it is the column itself, so the op is the window stage
    alone: window_flags (2 launches) + 3 per function (rank-like pass, SUM, COUNT) + the SUM column's validity pack"""
    n = 10_000
    rb = pa.RecordBatch.from_arrays([pa.array(np.repeat(np.arange(10), n // 10).astype(np.int64)), pa.array(np.arange(n, dtype=np.int64)),
                                     pa.array(np.arange(n, dtype=np.int64))], names=["p", "o", "v"])
    schema = T.Schema([T.Field(f, T.int64, False) for f in ("p", "o", "v")])
    exprs = [window_expr("rk", "rank", None, schema), window_expr("s", "sum", "v", schema), window_expr("c", "count", "v", schema)]
    plan = gpu_plan(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)])
    with native.NativeOp(plan.plan_bytes(), conf(**UNSTAGED)) as op:
        op.push(rb)
        op.finish()
        got = op.pull_all()
        m = op.metrics()
    assert m["gpu_kernel_launches"] == 2 + 3 * 3 + 1 and m["hot_kernel_rows"] == n
    osch, exp = oracle_run(schema, exprs, [E.Column("p")], [(E.Column("o"), False, True)], [rb])
    assert_equal_ordered(got, osch, exp)


def test_combining_rule_refuses_a_parent_without_window_columns():
    rb, schema = _limit_table()
    part, order = [E.Column("p")], [(E.Column("o"), False, True)]
    child = PL.WindowExec(PL.MemoryExec(schema), [window_expr("w", "rank", None, schema)], part, order, 3, False)
    parent = PL.WindowExec(child, [window_expr("rk", "row_number", None, schema)], part, order, None, False)
    with pytest.raises(native.NativeError) as ei:
        native.NativeOp(parent.plan_bytes())
    assert ei.value.code == native.ERR_UNSUPPORTED and "output_window_cols = false" in ei.value.msg
