"""An exact per-row reference for the expressions the device evaluates (FilterExec / ProjectExec, and the filters and
arguments fused into AggExec), written from the operations' definitions and sharing no code with the oracle.

Values are Python objects:
  None        NULL
  int         an integer of any width, a Boolean (0 / 1), or the unscaled value of a decimal128
  float       f64, and f32 as the exact f64 widening of the f32 value (every f32 is an f64)

Integers and decimals are Python ints, wrapped explicitly to the Rust width wherever the reference wraps (add / sub /
mul / neg wrapping, the CheckOverflow scale-up and its `dropped.abs() * 2`).  f64 operations are Python float
operations, each correctly rounded.  f32 `+ - * /` are computed in f64 and rounded once to f32: the f64 result of two f32
operands is exact or carries enough bits for that second rounding to be harmless; fmod is exact.  Integer -> float
rounds once, from the exact integer.  Decimal <-> float follow the formula the project assumes arrow uses:
`(v as f64) / 10^s` and `round(f * 10^s)` with halves away from zero, 10^s the correctly rounded f64 (exact up to
scale 22; above it the device's host-side `std::pow(10.0, s)` is assumed to agree, which test_exact_expr_reference.py
pins for this libm, and arrow's `powi` is assumed to agree as well, which nothing here can check).  Float comparisons
use IEEE totalOrder; float -> int follows Rust `as` (truncate, saturate, NaN -> 0).
"""
import math
import struct
from fractions import Fraction

from blaze_b200 import exprs as E, types as T

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
I128_MIN, I128_MAX = -(1 << 127), (1 << 127) - 1


class ArrowError(Exception):
    """an error the reference raises (kind: 'div_zero' | 'overflow')"""
    def __init__(self, kind):
        super().__init__(kind)
        self.kind = kind


# ---- integers -------------------------------------------------------------------------------------------------------------
def wrap(v: int, bits: int) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def int_range(bits: int):
    return -(1 << (bits - 1)), (1 << (bits - 1)) - 1


def add_wrapping(a, b, bits): return wrap(a + b, bits)
def sub_wrapping(a, b, bits): return wrap(a - b, bits)
def mul_wrapping(a, b, bits): return wrap(a * b, bits)
def neg_wrapping(a, bits): return wrap(-a, bits)


def _trunc_div(a: int, b: int) -> int:
    q = abs(a) // abs(b)
    return -q if (a < 0) != (b < 0) else q


def div_checked(a, b, bits):
    if b == 0:
        raise ArrowError("div_zero")
    if a == int_range(bits)[0] and b == -1:
        raise ArrowError("overflow")
    return _trunc_div(a, b)


def mod_checked(a, b, bits):
    if b == 0:
        raise ArrowError("div_zero")
    if a == int_range(bits)[0] and b == -1:
        raise ArrowError("overflow")
    return a - _trunc_div(a, b) * b                                   # the sign follows the dividend


# ---- binary floats -------------------------------------------------------------------------------------------------------
F64 = (53, -1022, 1023)      # (precision incl. the hidden bit, min normal exponent, max exponent)
F32 = (24, -126, 127)


def round_fraction(q, fmt) -> float:
    """the exact rational q rounded once to the binary format `fmt`, ties to even, overflow to ±inf"""
    p, emin, emax = fmt
    q = Fraction(q)
    if q == 0:
        return 0.0
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()          # 2^(e-1) < a < 2^(e+1)
    if Fraction(2) ** e > a:
        e -= 1                                                          # now 2^e <= a < 2^(e+1)
    e = max(e, emin)
    step = Fraction(2) ** (e - p + 1)                                   # the spacing of the format at a
    n, rem = divmod(a, step)
    if rem * 2 > step or (rem * 2 == step and n % 2):
        n += 1
    r = n * step
    if r >= Fraction(2) ** (emax + 1):
        return math.copysign(math.inf, q)
    return math.copysign(float(r), q)                                   # r is exact in f64


def to_f32(x: float) -> float:
    """`as f32` of an f64 value: ties to even, overflow to ±inf; NaN stays NaN"""
    if x != x or math.isinf(x) or x == 0:
        return x
    return round_fraction(Fraction(x), F32)


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f32_bits(x: float) -> int:
    """the f32 bit pattern of a non-NaN f32 value held as a Python float"""
    assert x == x
    return struct.unpack("<I", struct.pack("<f", x))[0]


def total_order_key(x: float) -> int:
    """IEEE totalOrder as an integer key (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN); f32 values order the same
    way as their f64 widenings, so one key serves both widths"""
    s = wrap(f64_bits(x), 64)
    return s ^ INT64_MAX if s < 0 else s


def _fdiv(a: float, b: float) -> float:
    if b == 0 or a != a or b != b:
        if a != a or b != b or a == 0:
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def _fmod(a: float, b: float) -> float:
    """C fmod / Rust `%`: exact; NaN for x = ±inf or y = 0; x itself for a finite x and y = ±inf"""
    if a != a or b != b or math.isinf(a) or b == 0:
        return math.nan
    if math.isinf(b):
        return a
    return math.fmod(a, b)


def float_arith(op: str, a: float, b: float, width: int) -> float:
    if op == "Plus": v = a + b
    elif op == "Minus": v = a - b
    elif op == "Multiply": v = a * b
    elif op == "Divide": v = _fdiv(a, b)
    else: v = _fmod(a, b)
    return to_f32(v) if width == 32 else v


def float_to_int(x: float, bits: int) -> int:
    """Rust `x as iN`: truncate toward zero, saturate, NaN -> 0"""
    lo, hi = int_range(bits)
    if x != x:
        return 0
    if math.isinf(x):
        return hi if x > 0 else lo
    return min(hi, max(lo, int(x)))                                     # int() truncates toward zero


def int_to_float(v: int, width: int) -> float:
    """`v as f64` / `v as f32`: one rounding of the exact integer"""
    return round_fraction(v, F64 if width == 64 else F32)


# ---- decimal128 ----------------------------------------------------------------------------------------------------------
def pow10_f64(s: int) -> float:
    return float(10 ** s)                                               # correctly rounded; exact for s <= 22


def round_half_away(q: Fraction) -> int:
    n = math.floor(abs(q) + Fraction(1, 2))
    return -n if q < 0 else n


def in_precision(v: int, precision: int) -> bool:
    lim = 10 ** precision
    return -lim < v < lim


def dec_to_float(v: int, scale: int, width: int) -> float:
    """(v as f64) / 10^s, then `as f32` for a Float32 result"""
    d = float(v) / pow10_f64(scale)                                     # float(int) rounds once, ties to even
    return to_f32(d) if width == 32 else d


def float_to_dec(x: float, precision: int, scale: int):
    """round(x * 10^s) with halves away from zero; NULL when not finite, beyond i128 or beyond the precision"""
    f = x * pow10_f64(scale)
    if not math.isfinite(f):
        return None
    v = round_half_away(Fraction(f))
    if not (I128_MIN < v < 1 << 127) or not in_precision(v, precision):   # double_to_i128 refuses |f| >= 2^127
        return None
    return v


def int_to_dec(v: int, precision: int, scale: int):
    v *= 10 ** scale
    return v if in_precision(v, precision) and I128_MIN <= v <= I128_MAX else None


def dec_to_dec(v: int, frm, to):
    """arrow-cast decimal -> decimal (safe): halves away from zero when the scale drops, a checked multiply when it grows,
    NULL outside the target precision"""
    if to.scale < frm.scale:
        f = 10 ** (frm.scale - to.scale)
        q, rem = divmod(abs(v), f)
        if rem * 2 >= f:
            q += 1
        v = -q if v < 0 else q
    elif to.scale > frm.scale:
        v *= 10 ** (to.scale - frm.scale)
        if not I128_MIN <= v <= I128_MAX:
            return None
    return v if in_precision(v, to.precision) else None


def dec_to_int(v: int, scale: int, bits: int):
    q = _trunc_div(v, 10 ** scale)
    lo, hi = int_range(bits)
    return q if lo <= q <= hi else None


def check_overflow(v: int, frm, to):
    """Spark Decimal.changePrecision as the reference implements it (spark_check_overflow.rs:84-124), with the i128 wrapping
    of a release build: the scale-up multiply wraps, and so does `dropped.abs() * 2`, which turns negative (no rounding)
    once |dropped| >= 2^126"""
    if (to.precision, to.scale) == (frm.precision, frm.scale):
        return v
    if to.scale < frm.scale:
        f = 10 ** (frm.scale - to.scale)
        q = _trunc_div(v, f)
        dropped = v - q * f
        if wrap(abs(dropped) * 2, 128) >= f:
            q += -1 if dropped < 0 else 1
        v = q
    elif to.scale > frm.scale:
        v = wrap(v * 10 ** (to.scale - frm.scale), 128)
    return v if in_precision(v, min(to.precision, 38)) else None


def dec_add_checked(op: str, a: int, b: int, at, bt, rt) -> int:
    """arrow-arith decimal Add / Sub: both sides rescaled to the result scale, checked i128 arithmetic.  A result beyond the
    result precision that still fits i128 is returned as it is"""
    a *= 10 ** (rt.scale - at.scale)
    b *= 10 ** (rt.scale - bt.scale)
    v = a + b if op == "Plus" else a - b
    if not (I128_MIN <= a <= I128_MAX and I128_MIN <= b <= I128_MAX and I128_MIN <= v <= I128_MAX):
        raise ArrowError("overflow")
    return v


# ---- casts ----------------------------------------------------------------------------------------------------------------
def _intlike(t):
    return t.is_integer or t.id in (T.DATE32, T.TIMESTAMP_US)


def _bits(t):
    return {T.INT8: 8, T.INT16: 16, T.INT32: 32, T.DATE32: 32, T.INT64: 64, T.TIMESTAMP_US: 64}[t.id]


def _fwidth(t):
    return 32 if t.id == T.FLOAT32 else 64


def cast(v, frm, to):
    """Cast / TryCast of one non-NULL value (arrow-cast with safe options, float -> int by Rust `as`)"""
    if frm == to:
        return v
    if _intlike(frm) and _intlike(to):
        lo, hi = int_range(_bits(to))
        return v if lo <= v <= hi else None
    if frm.id == T.BOOL and to.is_integer:
        return v
    if (_intlike(frm) or frm.id == T.BOOL) and to.is_float:
        return int_to_float(v, _fwidth(to))
    if frm.is_float and to.is_integer:
        return float_to_int(v, _bits(to))
    if frm.is_float and to.is_float:
        return to_f32(v) if to.id == T.FLOAT32 else v
    if (frm.is_integer or frm.is_float) and to.id == T.BOOL:
        return int(v != 0)
    if frm.is_integer and to.is_decimal:
        return int_to_dec(v, to.precision, to.scale)
    if frm.is_decimal and to.is_decimal:
        return dec_to_dec(v, frm, to)
    if frm.is_decimal and to.is_integer:
        return dec_to_int(v, frm.scale, _bits(to))
    if frm.is_decimal and to.is_float:
        return dec_to_float(v, frm.scale, _fwidth(to))
    if frm.is_float and to.is_decimal:
        return float_to_dec(v, to.precision, to.scale)
    raise NotImplementedError(f"cast {frm} -> {to}")


# ---- comparisons ----------------------------------------------------------------------------------------------------------
def compare(op: str, a, b, t) -> int:
    if t.is_float:
        a, b = total_order_key(a), total_order_key(b)
    return int({"Eq": a == b, "NotEq": a != b, "Lt": a < b, "LtEq": a <= b, "Gt": a > b, "GtEq": a >= b}[op])


# ---- one expression over one row ------------------------------------------------------------------------------------------
def evaluate(e, row: dict, schema):
    """the value of expression `e` over `row` ({column name: value}); raises ArrowError where the reference errors"""
    t = e.data_type(schema)
    if isinstance(e, E.Column):
        return row[e.name]
    if isinstance(e, E.Literal):
        return e.value if e.value is None or not isinstance(e.value, bool) else int(e.value)
    if isinstance(e, (E.Cast, E.TryCast)):
        v = evaluate(e.expr, row, schema)
        return None if v is None else cast(v, e.expr.data_type(schema), t)
    if isinstance(e, E.Negative):
        v = evaluate(e.expr, row, schema)
        if v is None:
            return None
        if t.is_float:
            return -v
        return neg_wrapping(v, 128 if t.is_decimal else _bits(t))
    if isinstance(e, E.IsNull):
        return int(evaluate(e.expr, row, schema) is None)
    if isinstance(e, E.IsNotNull):
        return int(evaluate(e.expr, row, schema) is not None)
    if isinstance(e, E.Not):
        v = evaluate(e.expr, row, schema)
        return None if v is None else int(not v)
    if isinstance(e, E.BinaryExpr):
        return _binary(e, row, schema)
    if isinstance(e, E.InList):
        x = evaluate(e.expr, row, schema)
        xt = e.expr.data_type(schema)
        items = [evaluate(i, row, schema) for i in e.list]
        if x is None:
            return None
        found = any(i is not None and compare("Eq", x, i, xt) for i in items)
        if not found and any(i is None for i in items):
            return None
        return int(found != e.negated)
    if isinstance(e, E.Case):
        base = None if e.expr is None else evaluate(e.expr, row, schema)
        for w, th in e.when_then:
            wv = evaluate(w, row, schema)
            hit = (base is not None and wv is not None and compare("Eq", base, wv, e.expr.data_type(schema))) if e.expr is not None else bool(wv)
            if hit:
                return evaluate(th, row, schema)
        return None if e.else_expr is None else evaluate(e.else_expr, row, schema)
    if isinstance(e, E.ScalarFunction):
        a = evaluate(e.args[0], row, schema)
        at = e.args[0].data_type(schema)
        if a is None:
            return None
        if e.name == "UnscaledValue":
            return wrap(a, 64)
        if e.name == "MakeDecimal":
            return a
        if e.name == "CheckOverflow":
            return check_overflow(a, at, t)
        if e.name == "NullIfZero":
            return None if a == 0 else a
    raise NotImplementedError(repr(e))


def _binary(e, row, schema):
    op = e.op
    lt = e.left.data_type(schema)
    if op in ("And", "Or"):
        a, b = evaluate(e.left, row, schema), evaluate(e.right, row, schema)
        if op == "And":
            return 0 if a == 0 or b == 0 else (None if a is None or b is None else 1)
        return 1 if a == 1 or b == 1 else (None if a is None or b is None else 0)
    a, b = evaluate(e.left, row, schema), evaluate(e.right, row, schema)
    if a is None or b is None:
        return None
    if op in E.COMPARISONS:
        return compare(op, a, b, lt)
    if lt.is_decimal:
        return dec_add_checked(op, a, b, lt, e.right.data_type(schema), e.data_type(schema))
    if lt.is_float:
        return float_arith(op, a, b, _fwidth(lt))
    bits = _bits(lt)
    return {"Plus": add_wrapping, "Minus": sub_wrapping, "Multiply": mul_wrapping, "Divide": div_checked, "Modulo": mod_checked}[op](a, b, bits)


def same_value(exp, got, t, nan_bits=False) -> bool:
    """got: the engine's value (Python int / float, None for NULL).  Floats compare by bits at the type's width; a NaN by
    NaN-ness only unless nan_bits (then both are f64 bit patterns or f32 bit patterns given as ints)"""
    if exp is None or got is None:
        return exp is None and got is None
    if t.is_float:
        if exp != exp:
            return got != got
        if got != got:
            return False
        return (f32_bits(exp) == f32_bits(got)) if t.id == T.FLOAT32 else (f64_bits(exp) == f64_bits(got))
    return int(exp) == int(got)
