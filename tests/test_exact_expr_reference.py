"""The exact expression reference of tests/exact_expr.py against the reference's known answers (tests/kat_cases.py), against
hand-worked values at the numeric edges, and against the numpy oracle on random data away from the edges.  CPU only.

Decimal <-> float at scales above 22 rests on an assumption: 10^s is taken as the correctly rounded f64, which the device
now computes from the exact integer.  Arrow's `10_f64.powi(s)` is assumed to agree; a square-and-multiply powi would not
at scales 33, 34 and 37 (pinned below), and nothing here can check what arrow's build does."""
import math
import struct
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, types as T
from oracle import blaze_oracle as O
import exact_expr as X
import kat_cases

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _col_values(arr: pa.Array):
    """Python values of an arrow column (decimals unscaled)"""
    if pa.types.is_decimal(arr.type):
        words = arr.buffers()[1].to_pybytes()
        return [None if not arr[i].is_valid else int.from_bytes(words[(arr.offset + i) * 16:(arr.offset + i + 1) * 16], "little", signed=True)
                for i in range(len(arr))]
    return arr.to_pylist()


@pytest.mark.parametrize("case", kat_cases.cases(), ids=lambda c: c[0])
def test_reference_kats(case):
    name, _, inp, expr, exp = case
    schema = T.Schema([T.Field("x", T.from_arrow_type(inp.type), True)])
    dt = expr.data_type(schema)
    got = [X.evaluate(expr, {"x": v}, schema) for v in _col_values(inp)]
    want = _col_values(exp)
    assert all(X.same_value(w, g, dt) for w, g in zip(want, got)), f"{name}: {got} != {want}"


# ---- hand-worked values -------------------------------------------------------------------------------------------------
def test_float_to_decimal_rounds_halves_away_from_zero_exactly():
    # 0.49999999999999994 + 0.5 rounds to 1.0 in f64; f64::round gives 0
    assert X.float_to_dec(0.49999999999999994, 38, 0) == 0
    assert X.float_to_dec(-0.49999999999999994, 38, 0) == 0
    assert X.float_to_dec(2.0 ** 52 + 1, 38, 0) == 2 ** 52 + 1            # + 0.5 would round to even (2^52 + 2)
    assert X.float_to_dec(2.5, 38, 0) == 3 and X.float_to_dec(-2.5, 38, 0) == -3
    assert X.float_to_dec(0.5, 38, 0) == 1 and X.float_to_dec(-0.5, 38, 0) == -1
    assert X.float_to_dec(1.5e38, 38, 0) is None and X.float_to_dec(math.inf, 38, 0) is None and X.float_to_dec(math.nan, 10, 2) is None
    assert X.float_to_dec(2.0 ** 127, 38, 0) is None                       # beyond i128 (and the precision)


def test_oracle_float_to_decimal_matches_at_the_halfway_values():
    vals = [0.49999999999999994, -0.49999999999999994, 2.0 ** 52 + 1, -(2.0 ** 52 + 1), 2.5, -2.5, 4503599627370497.0]
    c = O.cast(O.Col(T.float64, np.array(vals), np.ones(len(vals), bool)), T.decimal128(38, 0))
    assert [int(v) for v in c.values] == [X.float_to_dec(v, 38, 0) for v in vals]


def test_check_overflow_wraps_the_doubled_remainder():
    frm, to = T.decimal128(38, 38), T.decimal128(38, 0)
    for v, want in [(9 * 10 ** 37, 0), (-9 * 10 ** 37, 0),                  # |dropped| >= 2^126: the i128 product wraps, no rounding
                    (8 * 10 ** 37, 1), (-8 * 10 ** 37, -1),                  # below 2^126: rounds half up
                    (5 * 10 ** 37, 1), (5 * 10 ** 37 - 1, 0), (10 ** 38 - 1, 0)]:
        assert X.check_overflow(v, frm, to) == want, v
        assert O.change_precision_round_half_up(v, 38, 38, 38, 0) == want, v
    assert X.check_overflow(1 << 126, frm, to) == 0 and X.check_overflow((1 << 126) - 1, frm, to) == 1
    # the scale-up multiply wraps before the precision check
    assert X.check_overflow(10 ** 20, T.decimal128(38, 0), T.decimal128(38, 20)) is None
    assert X.check_overflow(12345, T.decimal128(10, 2), T.decimal128(10, 2)) == 12345
    assert X.check_overflow(15, T.decimal128(10, 1), T.decimal128(10, 0)) == 2 and X.check_overflow(-15, T.decimal128(10, 1), T.decimal128(10, 0)) == -2


def test_int_to_float_rounds_once():
    v = 2 ** 62 + 2 ** 38 + 1
    assert X.int_to_float(v, 32) == 2.0 ** 62 + 2.0 ** 39
    assert struct.unpack("<f", struct.pack("<f", float(v)))[0] == 2.0 ** 62       # the double rounding a careless reference does
    assert X.int_to_float(v, 32) == float(np.float32(np.int64(v)))
    assert X.int_to_float(2 ** 53 + 1, 64) == 2.0 ** 53 and X.int_to_float(2 ** 53 + 3, 64) == 2.0 ** 53 + 4
    assert X.int_to_float(I64_MAX, 64) == 2.0 ** 63 and X.int_to_float(I64_MIN, 32) == -(2.0 ** 63)
    assert X.int_to_float(16777217, 32) == 16777216.0 and X.int_to_float(16777219, 32) == 16777220.0


def test_float_to_int_truncates_saturates_and_zeroes_nan():
    for bits in (8, 16, 32, 64):
        lo, hi = X.int_range(bits)
        assert X.float_to_int(math.nan, bits) == 0 and X.float_to_int(-math.nan, bits) == 0
        assert X.float_to_int(math.inf, bits) == hi and X.float_to_int(-math.inf, bits) == lo
        assert X.float_to_int(float(hi) + 1.0, bits) == hi and X.float_to_int(float(lo) - 1.0, bits) == lo
        assert X.float_to_int(-0.9, bits) == 0 and X.float_to_int(-1.9, bits) == -1 and X.float_to_int(2.5, bits) == 2
    assert X.float_to_int(9.2e18, 64) == 9200000000000000000 and X.float_to_int(2.0 ** 63, 64) == I64_MAX
    assert X.float_to_int(127.99, 8) == 127 and X.float_to_int(-128.99, 8) == -128


def test_wrapping_and_checked_integer_arithmetic():
    for bits in (8, 16, 32, 64):
        lo, hi = X.int_range(bits)
        assert X.add_wrapping(hi, 1, bits) == lo and X.sub_wrapping(lo, 1, bits) == hi
        assert X.neg_wrapping(lo, bits) == lo and X.mul_wrapping(lo, -1, bits) == lo
        for op in (X.div_checked, X.mod_checked):
            with pytest.raises(X.ArrowError) as ei:
                op(lo, -1, bits)
            assert ei.value.kind == "overflow"
            with pytest.raises(X.ArrowError) as ei:
                op(1, 0, bits)
            assert ei.value.kind == "div_zero"
        assert X.div_checked(lo, 1, bits) == lo and X.mod_checked(lo, -2, bits) == 0
    assert X.mul_wrapping(3037000499, 3037000499, 64) == 3037000499 ** 2
    assert X.mul_wrapping(3037000500, 3037000500, 64) == 3037000500 ** 2 - 2 ** 64
    assert X.div_checked(-7, 2, 64) == -3 and X.mod_checked(-7, 2, 64) == -1 and X.mod_checked(7, -2, 64) == 1


def test_f32_arithmetic_rounds_once_and_ieee_specials():
    a, b = X.to_f32(16777216.0), X.to_f32(1.0)
    assert X.float_arith("Plus", a, b, 32) == 16777216.0                    # ties to even
    assert X.float_arith("Plus", a, 3.0, 32) == 16777220.0
    assert X.float_arith("Multiply", 3.4028234663852886e38, 2.0, 32) == math.inf
    assert X.float_arith("Divide", 1.0, 3.0, 32) == float(np.float32(1.0) / np.float32(3.0))
    assert X.float_arith("Divide", 1.0, -0.0, 64) == -math.inf and math.isnan(X.float_arith("Divide", 0.0, 0.0, 64))
    assert math.isnan(X.float_arith("Modulo", 1.0, 0.0, 64)) and math.isnan(X.float_arith("Modulo", math.inf, 2.0, 64))
    assert X.float_arith("Modulo", -5.5, math.inf, 64) == -5.5 and X.float_arith("Modulo", -7.0, 2.0, 64) == -1.0
    assert math.copysign(1.0, X.float_arith("Modulo", -4.0, 2.0, 64)) < 0
    assert X.to_f32(1e-46) == 0.0 and X.to_f32(1.5e-45) == 2.0 ** -149 and X.to_f32(3.4028235677973366e38) == math.inf


def test_to_f32_against_numpy_on_random_f64():
    rng = np.random.default_rng(3)
    xs = rng.normal(0, 1, 4000) * np.exp2(rng.integers(-160, 130, 4000))
    with np.errstate(over="ignore"):
        assert all(X.to_f32(float(x)) == float(np.float32(x)) for x in xs)


def test_round_fraction_is_correctly_rounded():
    for q in (Fraction(1, 3), Fraction(2, 3), Fraction(10) ** 23, Fraction(-7, 10), Fraction(1, 10 ** 300), Fraction(1, 10 ** 320)):
        assert X.round_fraction(q, X.F64) == float(q)                      # float(Fraction) rounds once


def test_total_order_comparisons():
    t = T.float64
    assert X.compare("Lt", -0.0, 0.0, t) and not X.compare("Eq", -0.0, 0.0, t)
    neg_nan = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]
    assert X.compare("Gt", math.nan, math.inf, t) and X.compare("Lt", neg_nan, -math.inf, t) and X.compare("Eq", math.nan, math.nan, t)


def test_decimal_to_float_and_powers_of_ten():
    assert X.dec_to_float(1, 1, 64) == 0.1 and X.dec_to_float(-(10 ** 38 - 1), 0, 64) == -1e38
    assert X.dec_to_float(10 ** 38 - 1, 38, 32) == 1.0
    assert all(X.pow10_f64(s) == 10.0 ** s for s in range(23))              # exact
    # square-and-multiply powi (compiler-rt __powidf2) differs from the correctly rounded power above scale 22 here:
    def powi(a, b):
        r = 1.0
        while True:
            if b & 1:
                r *= a
            b //= 2
            if b == 0:
                return r
            a *= a
    assert [s for s in range(39) if powi(10.0, s) != X.pow10_f64(s)] == [33, 34, 37]


def test_decimal_add_overflow_and_wide_results():
    d38 = T.decimal128(38, 0)
    assert X.dec_add_checked("Plus", 10 ** 38 - 1, 1, d38, d38, d38) == 10 ** 38               # beyond the precision, fits i128
    with pytest.raises(X.ArrowError):
        X.dec_add_checked("Plus", X.I128_MAX, 1, d38, d38, d38)
    with pytest.raises(X.ArrowError):
        X.dec_add_checked("Minus", X.I128_MIN, 1, d38, d38, d38)
    assert X.dec_add_checked("Plus", 5, 7, T.decimal128(10, 1), T.decimal128(10, 3), T.decimal128(13, 3)) == 507


def test_decimal_casts():
    d = T.decimal128
    assert X.dec_to_dec(15, d(10, 1), d(10, 0)) == 2 and X.dec_to_dec(-15, d(10, 1), d(10, 0)) == -2 and X.dec_to_dec(14, d(10, 1), d(10, 0)) == 1
    assert X.dec_to_dec(10 ** 37, d(38, 0), d(38, 2)) is None and X.dec_to_dec(10 ** 36, d(38, 0), d(38, 2)) is None
    assert X.dec_to_dec(10 ** 20, d(38, 0), d(38, 30)) is None                # the multiply overflows i128
    assert X.dec_to_int(-(2 ** 63) * 100 - 99, 2, 64) == -(2 ** 63) and X.dec_to_int((2 ** 63) * 100, 2, 64) is None
    assert X.int_to_dec(I64_MIN, 38, 18) == I64_MIN * 10 ** 18 and X.int_to_dec(I64_MAX, 20, 2) is None


# ---- against the oracle on random data away from the edges --------------------------------------------------------------
def test_against_the_oracle_away_from_the_edges():
    rng = np.random.default_rng(17)
    n = 2000
    a = rng.integers(-10 ** 6, 10 ** 6, n)
    b = rng.integers(1, 1000, n)
    f = rng.normal(0, 1e3, n)
    g = rng.normal(0, 10, n).astype(np.float32)
    dv = [int(x) for x in rng.integers(-10 ** 12, 10 ** 12, n)]
    rb = pa.RecordBatch.from_arrays([pa.array(a), pa.array(b), pa.array(f), pa.array(g), kat_cases.raw_decimal_array(dv, 20, 4)],
                                    names=["a", "b", "f", "g", "d"])
    schema = T.from_arrow_schema(rb.schema)
    A, B, F, G, D = (E.Column(c) for c in "abfgd")
    exprs = [E.BinaryExpr(A, "Multiply", B), E.BinaryExpr(A, "Divide", B), E.BinaryExpr(A, "Modulo", B), E.Negative(A),
             E.BinaryExpr(F, "Divide", E.TryCast(B, T.float64)), E.BinaryExpr(G, "Multiply", G), E.BinaryExpr(G, "Modulo", E.Literal(3.0, T.float32)),
             E.TryCast(F, T.int32), E.TryCast(F, T.decimal128(20, 3)), E.TryCast(A, T.float32), E.TryCast(A, T.int16),
             E.TryCast(D, T.float64), E.TryCast(D, T.decimal128(18, 1)), E.TryCast(D, T.int32), E.TryCast(D, T.decimal128(30, 8)),
             E.ScalarFunction("CheckOverflow", [D, E.Literal(12, T.int32), E.Literal(1, T.int32)], T.decimal128(12, 1)),
             E.BinaryExpr(D, "Plus", D), E.BinaryExpr(F, "Lt", E.Literal(0.0, T.float64)),
             E.InList(A, [E.Literal(int(a[0]), T.int64), E.Literal(None, T.int64)]),
             E.Case(None, [(E.BinaryExpr(A, "Gt", E.Literal(0, T.int64)), F)], E.Negative(F))]
    ob = O.batch_from_arrow(rb)
    rows = [{c: _col_values(rb.column(c))[r] for c in "abfgd"} for r in range(n)]
    for c in "fg":
        for r, v in zip(rows, rb.column(c).to_pylist()):
            r[c] = float(v)
    for e in exprs:
        dt = e.data_type(schema)
        oc = O.evaluate(e, ob).broadcast(n)
        oracle_vals = [None if not oc.valid[r] else (float(oc.values[r]) if dt.is_float else int(oc.values[r])) for r in range(n)]
        bad = [(r, w, g) for r, w, g in ((r, X.evaluate(e, rows[r], schema), oracle_vals[r]) for r in range(n)) if not X.same_value(w, g, dt)]
        assert not bad, f"{e}: {len(bad)} rows differ, e.g. {bad[:3]}"
