"""FilterExec / ProjectExec expressions on the GPU against the exact reference of tests/exact_expr.py, on columns built
from the numeric edges of int8..int64, f32 / f64 and decimal128, mixed with random filler and NULLs.

Every expression family of the device evaluator (vm.cuh) runs through the VM kernel (force_generic_kernels=1) and the
default dispatch, on staged and on direct input.  The lean FilterExec / ProjectExec kernel and the merged filter intervals
of the aggregate's specialised kernels are checked on their own edges, with their launches asserted.  Results compare bit
for bit; a NaN produced by arithmetic or a cast compares by NaN-ness, and a NaN that passes through unchanged by its bits.

Decimal <-> float casts above scale 22 rest on the assumption stated in tests/exact_expr.py (10^s is the correctly rounded
f64 on both sides)."""
import math
import struct

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
import exact_expr as X
from kat_cases import raw_decimal_array

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
WIDTHS = {8: T.int8, 16: T.int16, 32: T.int32, 64: T.int64}
CONFS = {"vm_direct": dict(staging_rows=0, force_generic_kernels=1), "vm_staged": dict(force_generic_kernels=1),
         "default_direct": dict(staging_rows=0), "default_staged": {}}


def f64_of_bits(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


# ---- edge sets ------------------------------------------------------------------------------------------------------------
def int_edges(bits):
    lo, hi = X.int_range(bits)
    vals = {lo, lo + 1, -1, 0, 1, hi - 1, hi, 2 ** 31 - 1, 2 ** 31 + 1, -(2 ** 31) - 1, 3037000499, 3037000500, -3037000500,
            2 ** 62 + 2 ** 38 + 1, 2 ** 53 + 1, 16777217}
    return sorted(v for v in vals if lo <= v <= hi)


F32_MAX = 3.4028234663852886e38
F64_NAN_PAYLOADS = [f64_of_bits(0x7FF8000000000456), f64_of_bits(0xFFF8000000000123)]


def float_edges():
    out = [0.0, -0.0, math.inf, -math.inf, math.nan, *F64_NAN_PAYLOADS, 5e-324, -5e-324, 2.2250738585072009e-308,
           1.7976931348623157e308, -1.7976931348623157e308, 0.49999999999999994, -0.49999999999999994, 0.5, 2.5, -2.5,
           2.0 ** 52 + 1, 2.0 ** 53 + 2, -(2.0 ** 53), F32_MAX, 1.401298464324817e-45, 1e-40, 123.456, -987.654, 1e20, 3.0]
    for bits in (8, 16, 32, 64):
        lo, hi = X.int_range(bits)
        out += [float(hi), float(lo), float(hi) + 1.0, float(lo) - 1.0, math.nextafter(float(lo), 0.0), math.nextafter(float(hi), 0.0)]
        if bits < 64:
            out += [hi + 0.5, lo - 0.5, hi + 0.99, lo - 0.99]
    return out


def dec_edges():
    out = []
    for p in (9, 18, 19, 38):
        out += [10 ** p - 1, -(10 ** p - 1)]
    out += [2 ** 64 // 10 ** 10, 2 ** 64 // 10 ** 10 + 1, 2 ** 127 // 10 ** 10, 2 ** 127 // 10 ** 10 + 1, 2 ** 64 - 1, 2 ** 64, -(2 ** 64),
            2 ** 63, -(2 ** 63) - 1, 2 ** 126, -(2 ** 126), 9 * 10 ** 37, -9 * 10 ** 37, 8 * 10 ** 37, 5 * 10 ** 37, -5 * 10 ** 37]
    for k in (1, 2, 10, 20, 37):
        h = 5 * 10 ** (k - 1)
        out += [12 * 10 ** k + h, -(12 * 10 ** k + h), 12 * 10 ** k + h - 1, -(12 * 10 ** k + h - 1), h, -h]
    out += [10 * 5, -50, 150, -150, 0, 1, -1]
    out += [2 ** 64 + 2 ** 11 + 1, -(2 ** 64 + 2 ** 11 + 1), ((2 ** 63 + 2 ** 10) << 60) + 1]   # i128 -> f64: a tie in the top 64 bits, broken by a low bit
    for bits in (8, 16, 32, 64):                                        # decimal -> int exactly at and past each width's ends
        lo, hi = X.int_range(bits)
        out += [lo, hi, lo - 1, hi + 1, lo * 100 - 99, hi * 100 + 99, lo * 10 ** 10, hi * 10 ** 18 + 10 ** 18 - 1]
    return [v for v in out if -(10 ** 38) < v < 10 ** 38]


# ---- columns and runs -----------------------------------------------------------------------------------------------------
def f32_array(vals, valid):
    """f32 column from Python floats; the NaN rows take f32 NaNs with a non-default payload, both signs"""
    bits = []
    for i, v in enumerate(vals):
        if v is None or not valid[i]:
            bits.append(0)
        elif v != v:
            bits.append(0x7FC00123 if i % 2 else 0xFFC00456)
        else:
            bits.append(X.f32_bits(X.to_f32(v)))
    arr = np.array(bits, np.uint32).view(np.float32)
    return pa.array(arr, mask=~np.array(valid)), [None if not valid[i] else float(arr[i]) for i in range(len(vals))]


def column(vals, dt):
    """(arrow array, reference values) of Python values (None = NULL)"""
    valid = [v is not None for v in vals]
    if dt.id == T.FLOAT32:
        return f32_array(vals, valid)
    if dt.is_decimal:
        return raw_decimal_array(vals, dt.precision, dt.scale), list(vals)
    return pa.array(vals, type=T.to_arrow_type(dt)), list(vals)


def pairs_table(rng, edges_a, edges_b, filler_a, filler_b, null_frac=0.08):
    """every (a, b) pair of the edge sets, then filler rows, shuffled, with NULLs on either side"""
    a = [x for x in edges_a for _ in edges_b] + filler_a
    b = [y for _ in edges_a for y in edges_b] + filler_b
    perm = rng.permutation(len(a))
    a, b = [a[i] for i in perm], [b[i] for i in perm]
    a = [None if rng.random() < null_frac else x for x in a]
    b = [None if rng.random() < null_frac else y for y in b]
    return a, b


def make_batch(cols):
    """cols: {name: (values, dtype)} -> (RecordBatch, rows as dicts of reference values)"""
    arrays, ref = [], {}
    for name, (vals, dt) in cols.items():
        arr, rv = column(vals, dt)
        arrays.append(arr)
        ref[name] = rv
    rb = pa.RecordBatch.from_arrays(arrays, names=list(cols))
    n = rb.num_rows
    return rb, [{c: ref[c][r] for c in cols} for r in range(n)]


def values_of(arr):
    if pa.types.is_decimal(arr.type):
        words = arr.buffers()[1].to_pybytes()
        return [None if not arr[i].is_valid else int.from_bytes(words[(arr.offset + i) * 16:(arr.offset + i + 1) * 16], "little", signed=True)
                for i in range(len(arr))]
    if pa.types.is_boolean(arr.type):
        return [None if v is None else int(v) for v in arr.to_pylist()]
    if pa.types.is_temporal(arr.type):
        arr = arr.view(pa.int64() if arr.type.bit_width == 64 else pa.int32())
    return arr.to_pylist()


def run(rb, filters, projs, cf, batch_rows=700):
    batches = [rb.slice(i, batch_rows) for i in range(0, rb.num_rows, batch_rows)]
    leaf = PL.MemoryExec.from_arrow(batches, rb.schema)
    plan = PL.FilterExec(filters, leaf) if filters else leaf
    plan = PL.ProjectExec([(e, f"o{i}") for i, e in enumerate(projs)], plan)
    out = PL.collect(plan, native.default_conf(**cf))
    tab = pa.Table.from_batches(out, schema=out[0].schema) if out else None
    return [values_of(tab.column(i).combine_chunks()) for i in range(len(projs))] if tab is not None else [[] for _ in projs], plan


def check(rb, rows, projs, cf, filters=(), chunk=16):
    schema = T.from_arrow_schema(rb.schema)
    keep = [r for r in rows if all(X.evaluate(f, r, schema) == 1 for f in filters)]
    bad = []
    for i in range(0, len(projs), chunk):
        part = projs[i:i + chunk]
        got, _ = run(rb, list(filters), part, cf)
        for e, g in zip(part, got):
            dt = e.data_type(schema)
            exp = [X.evaluate(e, r, schema) for r in keep]
            assert len(g) == len(exp), f"{e}: {len(g)} rows, expected {len(exp)}"
            for r, ev, gv in zip(keep, exp, g):
                if not X.same_value(ev, gv, dt):
                    bad.append((e, r, ev, gv))
    assert not bad, f"{len(bad)} values differ from the exact reference, e.g. " + "; ".join(f"{e} over {r}: expected {ev!r}, got {gv!r}" for e, r, ev, gv in bad[:5])


# ---- integers -------------------------------------------------------------------------------------------------------------
def int_case(bits):
    rng = np.random.default_rng(bits)
    lo, hi = X.int_range(bits)
    edges = int_edges(bits)
    divisors = [d for d in edges if d not in (0, -1)] + [7, -3]
    fa = [int(v) for v in rng.integers(lo, hi, 200, endpoint=True)]
    fb = [int(v) for v in rng.integers(lo, hi, 200, endpoint=True)]
    a, b = pairs_table(rng, edges, edges, fa, fb)
    d = [divisors[int(i)] for i in rng.integers(0, len(divisors), len(a))]
    dt = WIDTHS[bits]
    rb, rows = make_batch({"a": (a, dt), "b": (b, dt), "d": (d, dt)})
    A, B, D = E.Column("a"), E.Column("b"), E.Column("d")
    L = lambda v: E.Literal(v, dt)
    projs = [E.BinaryExpr(A, op, B) for op in ("Plus", "Minus", "Multiply")] + [E.Negative(A)]
    projs += [E.BinaryExpr(A, "Divide", D), E.BinaryExpr(A, "Modulo", D), E.BinaryExpr(A, "Multiply", L(hi)), E.BinaryExpr(L(lo), "Minus", A)]
    projs += [E.TryCast(A, t) for w, t in WIDTHS.items() if w != bits] + [E.TryCast(A, T.float32), E.TryCast(A, T.float64), E.TryCast(A, T.bool_)]
    projs += [E.TryCast(A, T.decimal128(p, s)) for p, s in ((38, 0), (38, 18), (20, 2), (10, 0), (3, 0), (19, 0))]
    projs += [E.BinaryExpr(A, op, B) for op in E.COMPARISONS] + [E.BinaryExpr(A, "Lt", L(lo)), E.BinaryExpr(L(hi), "GtEq", A), E.BinaryExpr(A, "Eq", L(lo))]
    projs += [E.InList(A, [L(lo), L(hi), L(0)]), E.InList(A, [L(lo), L(-1), L(None)], True), E.ScalarFunction("NullIfZero", [A], dt),
              E.Case(None, [(E.BinaryExpr(A, "Lt", L(0)), E.Negative(A)), (E.IsNull(A), B)], A)]
    if bits == 64:
        projs += [E.ScalarFunction("MakeDecimal", [A, E.Literal(18, T.int32), E.Literal(2, T.int32)], T.decimal128(18, 2)),
                  E.TryCast(A, T.timestamp_us)]
    return rb, rows, projs


@pytest.mark.parametrize("cf", list(CONFS))
@pytest.mark.parametrize("bits", [8, 16, 32, 64])
def test_integer_expressions(bits, cf):
    rb, rows, projs = int_case(bits)
    check(rb, rows, projs, CONFS[cf])


# ---- floats ---------------------------------------------------------------------------------------------------------------
def float_case(dt):
    rng = np.random.default_rng(5 if dt.id == T.FLOAT64 else 6)
    edges = float_edges()
    if dt.id == T.FLOAT32:
        edges = [X.to_f32(v) for v in edges]
    sel = edges[::2] + [math.nan, -0.0]
    fill = [float(v) for v in rng.normal(0, 1e3, 200)]
    x, y = pairs_table(rng, edges, sel, fill, [float(v) for v in rng.normal(0, 10, 200)])
    rb, rows = make_batch({"x": (x, dt), "y": (y, dt)})
    Xc, Y = E.Column("x"), E.Column("y")
    L = lambda v: E.Literal(v, dt)
    projs = [E.BinaryExpr(Xc, op, Y) for op in E.ARITHMETIC] + [E.Negative(Xc)]
    projs += [E.TryCast(Xc, t) for t in WIDTHS.values()] + [E.TryCast(Xc, T.bool_), E.TryCast(Xc, T.float32 if dt.id == T.FLOAT64 else T.float64)]
    projs += [E.TryCast(Xc, T.decimal128(38, s)) for s in (0, 2, 10, 18, 22, 23, 30, 38)] + [E.TryCast(Xc, T.decimal128(10, 2))]
    projs += [E.BinaryExpr(Xc, op, Y) for op in E.COMPARISONS]
    projs += [E.BinaryExpr(Xc, "Eq", L(0.0)), E.BinaryExpr(Xc, "Lt", L(-0.0)), E.BinaryExpr(Xc, "GtEq", L(math.nan)), E.BinaryExpr(L(math.inf), "Lt", Xc)]
    projs += [E.InList(Xc, [L(-0.0), L(math.nan)]), E.InList(Xc, [L(0.0), L(None)], True), E.ScalarFunction("NullIfZero", [Xc], dt),
              E.Case(None, [(E.BinaryExpr(Xc, "Lt", Y), Xc)], Y)]
    return rb, rows, projs


@pytest.mark.parametrize("cf", list(CONFS))
@pytest.mark.parametrize("width", [64, 32])
def test_float_expressions(width, cf):
    rb, rows, projs = float_case(T.float64 if width == 64 else T.float32)
    check(rb, rows, projs, CONFS[cf])


@pytest.mark.parametrize("cf", ["vm_direct", "default_staged"])
def test_nan_payloads_pass_through_unchanged(cf):
    """f32 / f64 NaNs of both signs with non-default payloads keep their bits through a filtered projection and CASE (an f64
    signalling NaN too; an f32 one would come out quiet, as the evaluator widens f32 values to f64)"""
    f32_bits = [0x7FC00123, 0xFFC00456, 0xFFC00001, 0x3F800000, 0x80000000, 0x7F800000]
    f64_bits = [0x7FF8000000000456, 0xFFF8000000000123, 0x7FF4000000000001, 0x3FF0000000000000, 0x8000000000000000, 0x7FF0000000000000]
    n = len(f32_bits) * 50
    a = np.array(f32_bits * 50, np.uint32)
    b = np.array(f64_bits * 50, np.uint64)
    k = np.arange(n, dtype=np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(a.view(np.float32)), pa.array(b.view(np.float64)), pa.array(k)], names=["f", "d", "k"])
    F, D, K = E.Column("f"), E.Column("d"), E.Column("k")
    keep = E.BinaryExpr(E.BinaryExpr(K, "Modulo", E.Literal(3, T.int64)), "NotEq", E.Literal(1, T.int64))
    projs = [F, D, E.Case(None, [(E.BinaryExpr(K, "GtEq", E.Literal(0, T.int64)), F)], E.Literal(0.0, T.float32)),
             E.Case(None, [(E.BinaryExpr(K, "GtEq", E.Literal(0, T.int64)), D)], E.Literal(0.0, T.float64))]
    leaf = PL.MemoryExec.from_arrow([rb], rb.schema)
    plan = PL.ProjectExec([(e, f"o{i}") for i, e in enumerate(projs)], PL.FilterExec([keep], leaf))
    tab = pa.Table.from_batches(PL.collect(plan, native.default_conf(**CONFS[cf])))
    rows = [i for i in range(n) if i % 3 != 1]
    want32, want64 = a[rows], b[rows]
    for c, want, w in ((0, want32, np.uint32), (1, want64, np.uint64), (2, want32, np.uint32), (3, want64, np.uint64)):
        got = tab.column(c).combine_chunks().to_numpy(zero_copy_only=False).view(w)
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, f"output {c}: {len(bad)} values changed bits, e.g. {[(hex(int(want[i])), hex(int(got[i]))) for i in bad[:4]]}"


# ---- decimal128 -----------------------------------------------------------------------------------------------------------
SCALED = [0, 1, 2, 9, 10, 18, 20, 22, 23, 30, 33, 34, 37, 38]


def dec_case():
    rng = np.random.default_rng(9)
    edges = dec_edges()
    fill = [int(v) for v in rng.integers(-10 ** 18, 10 ** 18, 200)]
    a, b = pairs_table(rng, edges, [1, -1, 0, 10 ** 37, -(10 ** 37), 5, 7 * 10 ** 37], fill, [int(v) for v in rng.integers(-1000, 1000, 200)])
    i64 = [None if v is None else X.wrap(v, 64) for v in a]
    cols = {"a0": (a, T.decimal128(38, 0)), "b0": (b, T.decimal128(38, 0)), "i": (i64, T.int64)}
    for s in SCALED:
        cols[f"s{s}"] = (a, T.decimal128(38, s))
    rb, rows = make_batch(cols)
    d = T.decimal128
    A0, B0, I = E.Column("a0"), E.Column("b0"), E.Column("i")
    S = lambda s: E.Column(f"s{s}")
    lit = lambda v, s: E.Literal(v, d(38, s))
    projs = [E.TryCast(S(10), d(38, 0)), E.TryCast(S(10), d(38, 2)), E.TryCast(S(10), d(20, 2)), E.TryCast(S(10), d(38, 20)),
             E.TryCast(S(10), d(38, 38)), E.TryCast(A0, d(38, 10)), E.TryCast(S(37), d(38, 0)), E.TryCast(S(38), d(38, 1)), E.TryCast(A0, d(19, 0))]
    projs += [E.TryCast(S(s), t) for s in (0, 2, 10, 18) for t in WIDTHS.values()]
    projs += [E.TryCast(S(s), t) for s in SCALED for t in (T.float64, T.float32)]
    co = lambda col, p, s: E.ScalarFunction("CheckOverflow", [col, E.Literal(p, T.int32), E.Literal(s, T.int32)], d(p, s))
    projs += [co(S(38), 38, 0), co(S(37), 38, 0), co(S(10), 20, 2), co(S(10), 38, 9), co(A0, 38, 10), co(S(10), 38, 12), co(S(10), 38, 10), co(S(1), 38, 0)]
    projs += [E.ScalarFunction("UnscaledValue", [S(2)], T.int64), E.ScalarFunction("MakeDecimal", [I, E.Literal(38, T.int32), E.Literal(4, T.int32)], d(38, 4)),
              E.ScalarFunction("NullIfZero", [A0], d(38, 0)), E.Negative(S(10))]
    projs += [E.BinaryExpr(A0, "Plus", B0), E.BinaryExpr(A0, "Minus", B0), E.BinaryExpr(A0, "Lt", B0), E.BinaryExpr(S(10), "Lt", lit(0, 10)),
              E.BinaryExpr(A0, "GtEq", lit(10 ** 38 - 1, 0)), E.InList(A0, [lit(10 ** 38 - 1, 0), lit(-(10 ** 18 - 1), 0), lit(None, 0)]),
              E.Case(None, [(E.BinaryExpr(A0, "Lt", lit(0, 0)), B0)], A0)]
    return rb, rows, projs


@pytest.mark.parametrize("cf", list(CONFS))
def test_decimal_expressions(cf):
    rb, rows, projs = dec_case()
    check(rb, rows, projs, CONFS[cf])


def test_float_to_decimal_scales_0_to_38():
    """f64 / f32 -> decimal128(38, s) for every scale, and decimal(38, s) -> f64 for every scale"""
    rng = np.random.default_rng(11)
    edges = [v for v in float_edges() if v == v and abs(v) < 1e39] + [float(v) for v in rng.normal(0, 1, 60) * np.exp2(rng.integers(-60, 60, 60))]
    rb, rows = make_batch({"x": (edges, T.float64), "g": (edges, T.float32), **{f"s{s}": ([X.float_to_dec(v, 38, 0) for v in edges], T.decimal128(38, s)) for s in range(0, 39, 2)}})
    projs = [E.TryCast(E.Column(c), T.decimal128(38, s)) for s in range(39) for c in ("x", "g")]
    projs += [E.TryCast(E.Column(f"s{s}"), T.float64) for s in range(0, 39, 2)]
    check(rb, rows, projs, CONFS["vm_direct"])


# ---- errors ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 16, 32, 64])
@pytest.mark.parametrize("generic", [0, 1])
def test_division_errors_only_on_evaluated_valid_rows(bits, generic):
    lo, _ = X.int_range(bits)
    dt = WIDTHS[bits]
    cf = native.default_conf(staging_rows=0, force_generic_kernels=generic)
    A, B, K = E.Column("a"), E.Column("b"), E.Column("k")
    for bad_a, bad_b, words in ((5, 0, "Divide by zero"), (lo, -1, None)):
        for op in ("Divide", "Modulo"):
            # the offending row is valid and not filtered: an error
            rb = pa.RecordBatch.from_arrays([pa.array([1, bad_a, 3], T.to_arrow_type(dt)), pa.array([1, bad_b, 2], T.to_arrow_type(dt)),
                                             pa.array([0, 1, 0], pa.int64())], names=["a", "b", "k"])
            plan = PL.ProjectExec([(E.BinaryExpr(A, op, B), "q")], PL.MemoryExec.from_arrow([rb]))
            with pytest.raises(native.NativeError) as ei:
                PL.collect(plan, cf)
            assert ei.value.code == native.ERR_EXECUTION and (words is None or words in str(ei.value))
            # removed by an earlier conjunct: never evaluated
            plan = PL.FilterExec([E.BinaryExpr(K, "Eq", E.Literal(0, T.int64)), E.BinaryExpr(E.BinaryExpr(A, op, B), "GtEq", E.Literal(0, dt))],
                                 PL.MemoryExec.from_arrow([rb]))
            assert sum(b.num_rows for b in PL.collect(plan, cf)) == 2
            # the divisor's or the dividend's row is NULL: no error, a NULL result
            for mask in ([False, True, False],):
                rbn = pa.RecordBatch.from_arrays([rb.column(0), pa.array([1, bad_b, 2], T.to_arrow_type(dt), mask=np.array(mask)), rb.column(2)], names=["a", "b", "k"])
                out = PL.collect(PL.ProjectExec([(E.BinaryExpr(A, op, B), "q")], PL.MemoryExec.from_arrow([rbn])), cf)
                assert pa.Table.from_batches(out).column(0).to_pylist()[1] is None


@pytest.mark.parametrize("generic", [0, 1])
def test_decimal_add_overflow_is_an_error(generic):
    cf = native.default_conf(staging_rows=0, force_generic_kernels=generic)
    big = 10 ** 38 - 1
    rb = pa.RecordBatch.from_arrays([raw_decimal_array([1, big, 2], 38, 0), raw_decimal_array([1, big, 3], 38, 0),
                                     raw_decimal_array([1, 1, 1], 38, 10), pa.array([0, 1, 0], pa.int64())], names=["a", "b", "c", "k"])
    A, B, C, K = (E.Column(c) for c in "abck")
    for e in (E.BinaryExpr(A, "Plus", B), E.BinaryExpr(E.Negative(A), "Minus", B), E.BinaryExpr(A, "Plus", C)):
        with pytest.raises(native.NativeError) as ei:
            PL.collect(PL.ProjectExec([(e, "s")], PL.MemoryExec.from_arrow([rb])), cf)
        assert ei.value.code == native.ERR_EXECUTION
        plan = PL.FilterExec([E.BinaryExpr(K, "Eq", E.Literal(0, T.int64)), E.IsNotNull(e)], PL.MemoryExec.from_arrow([rb]))
        assert sum(b.num_rows for b in PL.collect(plan, cf)) == 2


# ---- the lean kernel ------------------------------------------------------------------------------------------------------
def lean_block():
    rng = np.random.default_rng(12)
    edges = int_edges(64)
    a, b = pairs_table(rng, edges, edges, [int(v) for v in rng.integers(I64_MIN, I64_MAX, 3000)],
                       [int(v) for v in rng.integers(I64_MIN, I64_MAX, 3000)], null_frac=0.0)
    return a, b


LEAN_LITS = [I64_MIN, -1, 0, 1, I64_MAX, 3037000500]


def lean_exprs(lit):
    A, B = E.Column("a"), E.Column("b")
    L = E.Literal(lit, T.int64)
    projs = [A, E.BinaryExpr(A, "Plus", B), E.BinaryExpr(A, "Minus", B), E.BinaryExpr(A, "Multiply", B),
             E.BinaryExpr(A, "Plus", L), E.BinaryExpr(A, "Minus", L), E.BinaryExpr(A, "Multiply", L), B]
    filters = [E.BinaryExpr(A, "GtEq", L), E.BinaryExpr(E.Literal(I64_MAX, T.int64), "GtEq", B)]
    return filters, projs


@pytest.mark.parametrize("lit", LEAN_LITS)
@pytest.mark.parametrize("op", E.COMPARISONS)
def test_lean_kernel_at_the_edges(op, lit):
    a, b = lean_block()
    rb, rows = make_batch({"a": (a, T.int64), "b": (b, T.int64)})
    _, projs = lean_exprs(lit)
    A, L = E.Column("a"), E.Literal(lit, T.int64)
    for filters in ([E.BinaryExpr(A, op, L)], [E.BinaryExpr(L, op, A)]):
        schema = T.from_arrow_schema(rb.schema)
        keep = [r for r in rows if all(X.evaluate(f, r, schema) == 1 for f in filters)]
        got, plan = run(rb, filters, projs, dict(staging_rows=0), batch_rows=rb.num_rows)
        assert plan.last_metrics["fast_path_launches"] > 0, "the lean kernel must run"
        for e, g in zip(projs, got):
            exp = [X.evaluate(e, r, schema) for r in keep]
            assert g == exp, f"{filters[0]} / {e}: {sum(x != y for x, y in zip(g, exp))} of {len(exp)} differ"


def test_lean_kernel_two_pass_form():
    """one batch of more than 2^20 rows: the count / scan / apply form"""
    a, b = lean_block()
    reps = (1 << 20) // len(a) + 1
    rb1, rows = make_batch({"a": (a, T.int64), "b": (b, T.int64)})
    rb = pa.RecordBatch.from_arrays([pa.concat_arrays([rb1.column(i)] * reps) for i in range(2)], names=["a", "b"])
    assert rb.num_rows >= 1 << 20
    schema = T.from_arrow_schema(rb.schema)
    filters, projs = lean_exprs(-1)
    keep = [r for r in rows if all(X.evaluate(f, r, schema) == 1 for f in filters)]
    got, plan = run(rb, filters, projs, dict(staging_rows=0), batch_rows=rb.num_rows)
    assert plan.last_metrics["fast_path_launches"] > 0
    for e, g in zip(projs, got):
        exp = [X.evaluate(e, r, schema) for r in keep] * reps
        assert g == exp, f"{e}: {sum(x != y for x, y in zip(g, exp))} of {len(exp)} differ"


# ---- merged filter intervals of the aggregate's specialised kernels --------------------------------------------------------
COL_TYPES = {"int8": T.int8, "int32": T.int32, "int64": T.int64, "date32": T.date32}


def interval_cases(dt):
    bits = 8 if dt.id == T.INT8 else 64 if dt.id == T.INT64 else 32
    lo, hi = X.int_range(bits)
    C = E.Column("c")
    if dt.id == T.DATE32:                                                  # no date32 -> int64 cast: the literals clamp to date32
        W, L64 = (lambda: C), (lambda v: E.Literal(max(lo, min(hi, v)), dt))
    else:                                                                  # a widening cast is read as the column itself
        W, L64 = ((lambda: E.TryCast(C, T.int64)) if bits < 64 else (lambda: C)), (lambda v: E.Literal(v, T.int64))
    Lc = lambda v: E.Literal(v, dt)
    cases = {
        "lt_min": [E.BinaryExpr(W(), "Lt", L64(I64_MIN))],
        "gt_max": [E.BinaryExpr(W(), "Gt", L64(I64_MAX))],
        "whole_range": [E.BinaryExpr(W(), "GtEq", L64(I64_MIN)), E.BinaryExpr(W(), "LtEq", L64(I64_MAX))],
        "empty_intersection": [E.BinaryExpr(C, "Gt", Lc(5)), E.BinaryExpr(C, "Lt", Lc(3))],
        "le_max_ge_min": [E.BinaryExpr(L64(I64_MAX), "GtEq", W()), E.BinaryExpr(L64(I64_MIN), "LtEq", W())],
        "eq_min": [E.BinaryExpr(C, "Eq", Lc(lo))],
        "eq_max": [E.BinaryExpr(Lc(hi), "Eq", C)],
        "four": [E.BinaryExpr(C, "GtEq", Lc(lo + 1)), E.BinaryExpr(C, "LtEq", Lc(hi - 1)), E.BinaryExpr(C, "Gt", Lc(-100)), E.BinaryExpr(C, "Lt", Lc(100))],
        "ge_max": [E.BinaryExpr(C, "GtEq", Lc(hi))],
        "lt_lo_plus_1": [E.BinaryExpr(C, "Lt", Lc(lo + 1))],
    }
    if bits < 64 and dt.id != T.DATE32:
        cases.update({"gt_width": [E.BinaryExpr(W(), "Gt", L64(hi))], "ge_below_width": [E.BinaryExpr(W(), "GtEq", L64(lo - 1))],
                      "lt_width_min": [E.BinaryExpr(W(), "Lt", L64(lo))], "le_above_width": [E.BinaryExpr(W(), "LtEq", L64(hi + 1))],
                      "gt_below_width": [E.BinaryExpr(W(), "Gt", L64(lo - 1)), E.BinaryExpr(W(), "Lt", L64(hi + 1))]})
    return cases, lo, hi


def interval_table(dt, lo, hi):
    rng = np.random.default_rng(hi & 0xFFFF)
    n = 6000
    edges = [lo, lo + 1, -1, 0, 1, 3, 4, 5, hi - 1, hi, -100, 99, 100]
    c = [edges[int(i)] if rng.random() < 0.5 else int(rng.integers(lo, hi, endpoint=True)) for i in rng.integers(0, len(edges), n)]
    c = [None if rng.random() < 0.05 else v for v in c]
    k = [int(v) for v in rng.integers(0, 16, n)]
    v = [None if rng.random() < 0.05 else int(x) for x in rng.integers(-10 ** 12, 10 ** 12, n)]
    return make_batch({"k": (k, T.int64), "c": (c, dt), "v": (v, T.int64), "x": ([None if y is None else float(y) for y in v], T.float64)})


@pytest.mark.parametrize("generic", [0, 1])
@pytest.mark.parametrize("sum_type", ["int64", "float64"])
@pytest.mark.parametrize("ctype", list(COL_TYPES))
def test_fused_filter_intervals(ctype, sum_type, generic):
    """SUM(int64) takes the specialised hashed or dense kernels; SUM(f64) the wide tile kernel, which always reads the merged
    intervals.  The f64 values are integers whose sums are exact in any order"""
    dt = COL_TYPES[ctype]
    st = T.int64 if sum_type == "int64" else T.float64
    cases, lo, hi = interval_cases(dt)
    rb, rows = interval_table(dt, lo, hi)
    schema = T.from_arrow_schema(rb.schema)
    bad = []
    for name, filters in cases.items():
        leaf = PL.MemoryExec.from_arrow([rb.slice(i, 2000) for i in range(0, rb.num_rows, 2000)], rb.schema)
        ins = leaf.schema()
        g = [E.GroupingExpr("k", E.Column("k"))]
        mk = lambda mode, ch: [E.AggExpr("s", mode, PL.create_agg(E.AGG_SUM, ch, ins, st)),
                               E.AggExpr("n", mode, PL.create_agg(E.AGG_COUNT, ch, ins, T.int64))]
        arg = "v" if sum_type == "int64" else "x"
        partial = PL.AggExec(PL.HashAgg, g, mk(E.PARTIAL, [E.Column(arg)]), False, PL.FilterExec(filters, leaf))
        final = PL.AggExec(PL.HashAgg, g, mk(E.FINAL, [E.placeholder(st)]), False, partial)
        out = pa.Table.from_batches(PL.collect(final, native.default_conf(staging_rows=0, force_generic_kernels=generic)), schema=T.to_arrow_schema(final.schema()))
        got = {k: (s, c) for k, s, c in zip(*(out.column(i).to_pylist() for i in range(3)))}
        exp = {}
        for r in rows:
            if all(X.evaluate(f, r, schema) == 1 for f in filters):
                s, cnt = exp.get(r["k"], (None, 0))
                if r["v"] is not None:
                    s, cnt = X.wrap((s or 0) + r["v"], 64), cnt + 1
                exp[r["k"]] = (s, cnt)
        if sum_type == "float64":
            exp = {k: (None if s is None else float(s), c) for k, (s, c) in exp.items()}
        if got != exp:
            bad.append((name, len(got), len(exp), sorted(set(got.items()) ^ set(exp.items()))[:2]))
        m = final.last_metrics["fast_path_launches"]
        if generic:
            assert m == 0
        elif exp:
            assert m > 0, f"{name}: the specialised kernels must run"
    assert not bad, f"{len(bad)} conjunct sets differ: {bad}"
