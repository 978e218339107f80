"""FilterExec / ProjectExec on the GPU vs the oracle (bit-exact, ordered)."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
from oracle import blaze_oracle as O
from helpers import *

pytestmark = pytest.mark.gpu


def run_fp(rb, predicates, projections, batch_rows=10000, conf=None):
    batches = split_batches(rb, batch_rows)
    leaf = PL.MemoryExec.from_arrow(batches, rb.schema)
    plan = leaf
    if predicates:
        plan = PL.FilterExec(predicates, plan)
    if projections is not None:
        plan = PL.ProjectExec(projections, plan)
    got = PL.collect(plan, conf)
    ins = leaf.schema()
    ob = oracle_batches(batches)
    if projections is not None:
        exp = O.ProjectExec(projections, ins, predicates).execute(ob)
    else:
        exp = O.FilterExec(predicates, ins).execute(ob)
    assert_same_rows_ordered(got, exp, plan.schema())
    return got, plan


def m0_batch(n, seed=42, null_frac=0.0):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1000, n, dtype=np.int64)
    b = rng.integers(-2**31, 2**31, n, dtype=np.int64)
    return rb_from_cols(["a", "b"], [with_nulls(rng, a, null_frac), with_nulls(rng, b, null_frac)])


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
@pytest.mark.parametrize("n", [1, 31, 513, 100_003])
def test_m0_filter_project(n, null_frac):
    rb = m0_batch(n, 42, null_frac)
    A, B = E.Column("a"), E.Column("b")
    run_fp(rb, [E.BinaryExpr(A, "Lt", E.Literal(500, T.int64))], [(A, "a"), (E.BinaryExpr(A, "Plus", B), "c")])


@pytest.mark.parametrize("thr", [-1, 0, 10, 990, 1000])
def test_selectivities_and_empty_output(thr):
    rb = m0_batch(50_000, 7, 0.05)
    A = E.Column("a")
    run_fp(rb, [E.BinaryExpr(A, "Lt", E.Literal(thr, T.int64))], None)


def test_filter_only_multiple_conjuncts_and_large_single_batch():
    rb = m0_batch(1_000_000, 3, 0.1)
    A, B = E.Column("a"), E.Column("b")
    preds = [E.BinaryExpr(A, "GtEq", E.Literal(100, T.int64)), E.BinaryExpr(B, "Lt", E.Literal(0, T.int64)), E.IsNotNull(A)]
    run_fp(rb, preds, None, batch_rows=1_000_000, conf=native.default_conf(staging_rows=0))


def test_project_only_no_filter():
    rb = m0_batch(70_001, 5, 0.2)
    A, B = E.Column("a"), E.Column("b")
    run_fp(rb, [], [(E.BinaryExpr(A, "Multiply", B), "m"), (E.BinaryExpr(B, "Minus", A), "d"), (E.IsNull(B), "bn"),
                    (E.BinaryExpr(A, "Lt", B), "lt")])


def test_scalar_predicates():
    rb = m0_batch(10_000, 9)
    A = E.Column("a")
    got, _ = run_fp(rb, [E.Literal(True, T.bool_), E.BinaryExpr(A, "Lt", E.Literal(10, T.int64))], None)
    got, _ = run_fp(rb, [E.Literal(None, T.bool_)], None)
    assert sum(b.num_rows for b in got) == 0


def test_mixed_types_casts_case_inlist():
    n = 40_000
    rng = np.random.default_rng(11)
    i32 = with_nulls(rng, rng.integers(-1000, 1000, n, dtype=np.int32), 0.1)
    f64 = with_nulls(rng, rng.normal(0, 1e3, n), 0.1)
    i8 = pa.array(rng.integers(-128, 128, n, dtype=np.int8))
    d32 = pa.array(rng.integers(0, 20000, n, dtype=np.int32), type=pa.int32()).cast(pa.date32())
    f32 = pa.array(rng.normal(0, 10, n).astype(np.float32))
    rb = rb_from_cols(["i", "f", "s", "d", "g"], [i32, f64, i8, d32, f32])
    I, F, S, D, G = (E.Column(c) for c in "ifsdg")
    projs = [
        (E.TryCast(I, T.int64), "i64"),
        (E.TryCast(F, T.int32), "f2i"),
        (E.TryCast(I, T.int8), "i2i8"),
        (E.TryCast(I, T.float64), "i2f"),
        (E.BinaryExpr(F, "Multiply", E.TryCast(I, T.float64)), "fm"),
        (E.BinaryExpr(G, "Plus", G), "gg"),
        (E.Case(None, [(E.BinaryExpr(I, "Lt", E.Literal(0, T.int32)), E.Literal(-1, T.int32)),
                       (E.BinaryExpr(I, "Eq", E.Literal(0, T.int32)), E.Literal(0, T.int32))], E.Literal(1, T.int32)), "sign"),
        (E.InList(I, [E.Literal(1, T.int32), E.Literal(2, T.int32), E.Literal(None, T.int32)], False), "in"),
        (E.InList(S, [E.Literal(5, T.int8), E.Literal(-7, T.int8)], True), "notin"),
        (E.BinaryExpr(E.BinaryExpr(I, "Gt", E.Literal(5, T.int32)), "Or", E.IsNull(F)), "or"),
        (E.BinaryExpr(E.BinaryExpr(I, "Gt", E.Literal(5, T.int32)), "And", E.BinaryExpr(F, "Lt", E.Literal(0.0, T.float64))), "and"),
        (E.Not(E.BinaryExpr(F, "GtEq", E.Literal(1.5, T.float64))), "not"),
        (E.Negative(I), "neg"),
        (E.BinaryExpr(D, "Lt", E.Literal(10000, T.date32)), "dlt"),
        (E.ScalarFunction("NullIfZero", [I], T.int32), "niz"),
        (E.BinaryExpr(I, "Modulo", E.ScalarFunction("NullIfZero", [E.TryCast(S, T.int32)], T.int32)), "mod"),
    ]
    run_fp(rb, [E.BinaryExpr(I, "NotEq", E.Literal(7, T.int32))], projs)


def test_decimal_exprs():
    import decimal
    n = 5000
    rng = np.random.default_rng(13)
    raw = rng.integers(-10**9, 10**9, n)
    dec = pa.array([None if i % 17 == 0 else decimal.Decimal(int(v)).scaleb(-2) for i, v in enumerate(raw)], type=pa.decimal128(12, 2))
    rb = rb_from_cols(["x"], [dec])
    X = E.Column("x")
    d12 = T.decimal128(12, 2)
    projs = [
        (E.ScalarFunction("UnscaledValue", [X], T.int64), "u"),
        (E.ScalarFunction("MakeDecimal", [E.ScalarFunction("UnscaledValue", [X], T.int64), E.Literal(12, T.int32), E.Literal(2, T.int32)], d12), "md"),
        (E.ScalarFunction("CheckOverflow", [X, E.Literal(8, T.int32), E.Literal(1, T.int32)], T.decimal128(8, 1)), "co"),
        (E.BinaryExpr(X, "Plus", X), "pp"),
        (E.TryCast(X, T.decimal128(20, 4)), "up"),
        (E.TryCast(X, T.decimal128(10, 0)), "down"),
        (E.TryCast(X, T.int64), "toi"),
        (E.TryCast(X, T.float64), "tof"),
        (E.BinaryExpr(X, "Lt", E.Literal(0, d12)), "neg"),
    ]
    run_fp(rb, [E.IsNotNull(X)], projs, batch_rows=1000)


def test_divide_by_zero_is_an_error():
    rb = rb_from_cols(["a", "b"], [pa.array([1, 2, 3], pa.int64()), pa.array([1, 0, 2], pa.int64())])
    plan = PL.ProjectExec([(E.BinaryExpr(E.Column("a"), "Divide", E.Column("b")), "q")], PL.MemoryExec.from_arrow([rb]))
    with pytest.raises(native.NativeError) as ei:
        PL.collect(plan)
    assert ei.value.code == native.ERR_EXECUTION and "Divide by zero" in str(ei.value)
    # rows removed by an earlier conjunct are never evaluated (evaluate_selection)
    plan = PL.FilterExec([E.BinaryExpr(E.Column("b"), "NotEq", E.Literal(0, T.int64)),
                          E.BinaryExpr(E.BinaryExpr(E.Column("a"), "Divide", E.Column("b")), "Gt", E.Literal(0, T.int64))],
                         PL.MemoryExec.from_arrow([rb]))
    out = PL.collect(plan)
    assert sum(b.num_rows for b in out) == 2


@pytest.mark.parametrize("generic", [0, 1])
@pytest.mark.parametrize("thr", [-1, 0, 3, 500, 999, 1000])
def test_lean_kernel_selectivities(thr, generic):
    """non-null int64 inputs take the lean (bytecode-free) kernel; it must agree with the VM kernel and the oracle"""
    rb = m0_batch(300_007, 21, 0.0)
    A, B = E.Column("a"), E.Column("b")
    projs = [(A, "a"), (E.BinaryExpr(A, "Plus", B), "c"), (E.BinaryExpr(B, "Minus", E.Literal(7, T.int64)), "d"), (E.BinaryExpr(A, "Multiply", B), "m")]
    conf = native.default_conf(staging_rows=0, force_generic_kernels=generic)
    got, plan = run_fp(rb, [E.BinaryExpr(A, "Lt", E.Literal(thr, T.int64)), E.BinaryExpr(E.Literal(-2**40, T.int64), "LtEq", B)], projs, batch_rows=120_000, conf=conf)
    assert (plan.last_metrics["fast_path_launches"] > 0) == (generic == 0)


def test_lean_project_only_and_filter_only():
    rb = m0_batch(99_999, 22, 0.0)
    A, B = E.Column("a"), E.Column("b")
    _, plan = run_fp(rb, [], [(E.BinaryExpr(A, "Multiply", E.Literal(3, T.int64)), "x"), (B, "b")])
    assert plan.last_metrics["fast_path_launches"] > 0
    _, plan = run_fp(rb, [E.BinaryExpr(A, "GtEq", E.Literal(990, T.int64))], None)
    assert plan.last_metrics["fast_path_launches"] > 0


@pytest.mark.parametrize("n", [1 << 20, 3_000_037])
def test_lean_large_batch_forms(n):
    """batches of >= 2^20 rows take the order-free count / scan / apply form: ragged last tile, 3 input columns, conjuncts on
    two of them, every selectivity regime inside one batch (sorted run + random part)"""
    rng = np.random.default_rng(n)
    a = rng.integers(0, 1000, n, dtype=np.int64); a[: n // 4] = np.sort(a[: n // 4])
    b = rng.integers(-2**31, 2**31, n, dtype=np.int64)
    c = rng.integers(-5, 5, n, dtype=np.int64)
    rb = rb_from_cols(["a", "b", "c"], [a, b, c])
    A, B, C = E.Column("a"), E.Column("b"), E.Column("c")
    preds = [E.BinaryExpr(A, "GtEq", E.Literal(200, T.int64)), E.BinaryExpr(A, "LtEq", E.Literal(700, T.int64)), E.BinaryExpr(C, "NotEq", E.Literal(0, T.int64))]
    projs = [(B, "b"), (E.BinaryExpr(A, "Multiply", C), "ac"), (E.BinaryExpr(B, "Minus", A), "d")]
    got, plan = run_fp(rb, preds, projs, batch_rows=n, conf=native.default_conf(staging_rows=0))
    assert plan.last_metrics["fast_path_launches"] > 0 and plan.last_metrics["gpu_kernel_launches"] >= 1


@pytest.mark.parametrize("ncols", [1, 2, 4])
def test_lean_large_batch_column_counts_and_unaligned_slices(ncols):
    """1 / 2 / 4 input columns; a batch that starts one row into its buffers is 8- but not 16-byte aligned: the two-pass form
    gives the same rows either way"""
    n = (1 << 20) + 4321
    rng = np.random.default_rng(ncols)
    cols = [rng.integers(0, 1000, n + 1, dtype=np.int64) for _ in range(ncols)]
    names = ["a", "b", "c", "d"][:ncols]
    whole = rb_from_cols(names, cols)
    A = E.Column("a")
    preds = [E.BinaryExpr(A, "Lt", E.Literal(300, T.int64))] + ([E.BinaryExpr(E.Column(names[-1]), "GtEq", E.Literal(100, T.int64))] if ncols > 1 else [])
    projs = [(E.Column(c), c) for c in names] + [(E.BinaryExpr(A, "Plus", E.Column(names[-1])), "s")]
    for rb in (whole.slice(0, n), whole.slice(1, n)):
        got, plan = run_fp(rb, preds, projs, batch_rows=n, conf=native.default_conf(staging_rows=0))
        assert plan.last_metrics["fast_path_launches"] > 0
