"""An exact group-by reference for SUM / AVG / MIN / MAX / COUNT, and seeded generators of numeric-edge groups.

The reference works on Python values and shares no code with the oracle's accumulators.  Each aggregate of a group
evaluates to one of:
  None                  NULL
  int                   an exact integer: int64, or the unscaled value of a decimal128
  float / np.float32    exact bits (a NaN is compared by NaN-ness only: its sign and payload are not a contract)
  Interval              an inexact f64 SUM / AVG: every summation order lands inside [center - radius, center + radius]

f64 SUM is exact bits whenever IEEE addition is order-independent over the group: a NaN or +inf together with -inf (NaN),
one infinity sign, zeros only (-0.0 when every value is -0.0: the reference stores the first value and adds the rest), all
values multiples of one 2^e whose magnitudes add up to less than 2^(53+e) (every partial sum, in any order, is exact), or
values of one sign whose exact sum is at least 2 * DBL_MAX (±inf in any order).  Otherwise the sum lies within
gamma(n-1) * sum|x_i| of the exact sum for every summation tree (Higham, Accuracy and Stability of Numerical Algorithms,
§4.2), gamma(k) = k u / (1 - k u), u = 2^-53: that covers atomics, Partial -> Final and the exchange alike.

f64 / f32 MIN and MAX follow IEEE totalOrder (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN), the order the GPU
keeps; the result is one of the group's input bit patterns.
"""
import math
import struct
import sys
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import pyarrow as pa

from blaze_b200 import exprs as E, types as T

U = Fraction(1, 1 << 53)
DBL_MAX = sys.float_info.max
DBL_MIN = sys.float_info.min
SUBNORMAL_MIN = 5e-324
F32_MAX = float(np.finfo(np.float32).max)
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
_SCALE = 1074                                   # every finite f64 is an integer multiple of 2^-1074


def gamma(k: int) -> Fraction:
    return k * U / (1 - k * U)


@dataclass(frozen=True)
class Interval:
    center: Fraction
    radius: Fraction

    def __contains__(self, x: float) -> bool:
        return math.isfinite(x) and abs(Fraction(x) - self.center) <= self.radius


def wrap(v: int, bits: int) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f32_bits(x) -> int:
    return int(np.float32(x).view(np.uint32))


NEG_NAN = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]


def to_f32(x: float) -> np.float32:
    """np.float32 of x, keeping the sign of a NaN"""
    if x != x:
        return np.array([0xFFC00000 if math.copysign(1.0, x) < 0 else 0x7FC00000], np.uint32).view(np.float32)[0]
    return np.float32(x)


def total_order_key(bits: int, width: int) -> int:
    """IEEE totalOrder as a signed integer key at the value's own width: negative values (sign bit set, NaN included)
    have their magnitude bits flipped, so that -NaN sorts first and +NaN last"""
    s = wrap(bits, width)
    return s ^ ((1 << (width - 1)) - 1) if s < 0 else s


# ---- f64 SUM / AVG -------------------------------------------------------------------------------------------------------
def _scaled(x: float) -> int:
    """x * 2^1074, an exact integer"""
    n, d = x.as_integer_ratio()
    return n << (_SCALE - (d.bit_length() - 1))


def f64_sum(xs):
    """SUM over the valid f64 values `xs` (Python floats) of one group -> None | float | Interval"""
    if not xs:
        return None
    if any(x != x for x in xs):
        return math.nan
    pinf, ninf = math.inf in xs, -math.inf in xs
    if pinf and ninf:
        return math.nan
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    if all(x == 0 for x in xs):
        return -0.0 if all(math.copysign(1.0, x) < 0 for x in xs) else 0.0
    sc = [_scaled(x) for x in xs]
    exact, mag = sum(sc), sum(abs(v) for v in sc)
    if (all(v >= 0 for v in sc) or all(v <= 0 for v in sc)) and abs(exact) >= 2 * _scaled(DBL_MAX):
        return math.inf if exact > 0 else -math.inf
    e = min((v & -v).bit_length() - 1 for v in sc if v)                 # all values are multiples of 2^(e - 1074)
    if mag < 1 << (53 + e) and mag <= _scaled(DBL_MAX):
        return float(Fraction(exact, 1 << _SCALE)) if exact else 0.0   # exact in any order; a cancelled sum is +0.0
    return Interval(Fraction(exact, 1 << _SCALE), gamma(len(xs) - 1) * Fraction(mag, 1 << _SCALE))


def f64_avg(xs):
    s = f64_sum(xs)
    if s is None:
        return None
    c = len(xs)
    if isinstance(s, float):
        return s / c                                                    # one correctly rounded division; -0.0 / c == -0.0
    # |fl(s'/c) - S/c| <= |s' - S| / c + u |s'| / c  with  |s' - S| <= radius
    return Interval(s.center / c, s.radius / c + U * (abs(s.center) + s.radius) / c)


# ---- MIN / MAX -----------------------------------------------------------------------------------------------------------
def float_minmax(xs, fn, width):
    """MIN / MAX under IEEE totalOrder; xs: Python floats (width 64) or np.float32 (width 32)"""
    if not xs:
        return None
    bits = f64_bits if width == 64 else f32_bits
    pick = min if fn == E.AGG_MIN else max
    return pick(xs, key=lambda x: total_order_key(bits(x), width))


def int_minmax(xs, fn):
    return None if not xs else (min(xs) if fn == E.AGG_MIN else max(xs))


# ---- decimal128 ----------------------------------------------------------------------------------------------------------
def dec_try_cast(v: int, frm, to):
    """TryCast of an unscaled decimal128 to a type of at least its scale: NULL when it overflows the target precision;
    the identical type is no cast at all"""
    if (frm.precision, frm.scale) == (to.precision, to.scale):
        return v
    v *= 10 ** (to.scale - frm.scale)
    return v if -10 ** to.precision < v < 10 ** to.precision else None


def dec_sum(vals, frm, to):
    cast = [c for c in (dec_try_cast(v, frm, to) for v in vals) if c is not None]
    return None if not cast else wrap(sum(cast), 128)


def dec_avg(vals, frm, to):
    cast = [c for c in (dec_try_cast(v, frm, to) for v in vals) if c is not None]
    return None if not cast else wrap(sum(cast), 128) // len(cast)     # div_euclid by a positive count


# ---- one aggregate over the valid values of one group --------------------------------------------------------------------
def aggregate(fn, arg_type, result_type, vals):
    """vals: the group's argument values, None for NULL (decimals unscaled, f32 as np.float32)"""
    valid = [v for v in vals if v is not None]
    if fn == E.AGG_COUNT:
        return len(valid)
    if fn in (E.AGG_MIN, E.AGG_MAX):
        if arg_type.id == T.FLOAT64:
            return float_minmax(valid, fn, 64)
        if arg_type.id == T.FLOAT32:
            return float_minmax(valid, fn, 32)
        return int_minmax(valid, fn)
    if arg_type.is_decimal:
        return (dec_sum if fn == E.AGG_SUM else dec_avg)(valid, arg_type, result_type)
    if result_type.id == T.FLOAT64:
        xs = [float(v) for v in valid]                                  # `as f64` of an integer: round to nearest even
        return (f64_sum if fn == E.AGG_SUM else f64_avg)(xs)
    assert fn == E.AGG_SUM and result_type.id == T.INT64
    return None if not valid else wrap(sum(valid), 64)


def expected_groups(keys, cols, specs, types):
    """{key tuple: [expected per spec]} of a GROUP BY over rows (keys[r] a tuple, cols[name][r] a value or None)"""
    rows = {}
    for r, k in enumerate(keys):
        rows.setdefault(k, []).append(r)
    out = {}
    for k, rs in rows.items():
        out[k] = [aggregate(fn, types[col] if col else None, rt, [cols[col][r] for r in rs] if col else [1] * len(rs))
                  for _, fn, col, rt in specs]
    return out


def matches(exp, got) -> bool:
    """got: None or the value the engine returned (Python float / np.float32 / int)"""
    if exp is None or got is None:
        return exp is None and got is None
    if isinstance(exp, Interval):
        return isinstance(got, float) and got in exp
    if isinstance(exp, (float, np.floating)):
        if exp != exp:
            return got != got
        if isinstance(exp, np.float32):
            return f32_bits(got) == f32_bits(exp)
        return f64_bits(float(got)) == f64_bits(exp)
    return int(got) == exp


# ---- generators ----------------------------------------------------------------------------------------------------------
# A family builds groups of (kind, [argument values]); `table` lays them out as rows of int64 key `k` + argument columns.
D38_0, D38_10, D38_2, D20_2 = T.decimal128(38, 0), T.decimal128(38, 10), T.decimal128(38, 2), T.decimal128(20, 2)
BIG = 10 ** 38 - 1


def f64_sum_groups(rng, ngroups=600):
    """edge groups of f64 SUM / AVG"""
    kinds = ["neg_zero", "neg_zero_nulls", "mixed_zeros", "pinf", "ninf", "pinf_ninf", "nan", "overflow", "subnormal",
             "dyadic", "dyadic_small_row", "ill_conditioned", "normal", "all_null"]
    out = []
    for g in range(ngroups):
        kind = kinds[g % len(kinds)]
        n = int(rng.integers(1, 6))
        fin = lambda m: [float(v) for v in rng.normal(0, 1e3, m)]
        if kind == "neg_zero":
            v = [-0.0] * n
        elif kind == "neg_zero_nulls":
            v = [-0.0] * n + [None] * int(rng.integers(1, 4))
        elif kind == "mixed_zeros":
            v = [-0.0] * n + [0.0]
        elif kind == "pinf":
            v = fin(n) + [math.inf]
        elif kind == "ninf":
            v = fin(n) + [-math.inf, -math.inf]
        elif kind == "pinf_ninf":
            v = fin(n) + [math.inf, -math.inf]
        elif kind == "nan":
            v = fin(n) + [math.nan]
        elif kind == "overflow":
            v = [1.5e308 * (1 if g % 2 else -1)] * 3                     # 4.5e308 >= 2 * DBL_MAX: ±inf in any order
        elif kind == "subnormal":
            v = [float(m) * SUBNORMAL_MIN * (1 if rng.random() < 0.5 else -1) for m in rng.integers(1, 1 << 40, n + 2)]
        elif kind == "dyadic":
            m = int(rng.integers(50, 400))
            v = [float(a) + float(b) / 4 for a, b in zip(rng.integers(-2 ** 40, 2 ** 40, m), rng.integers(0, 4, m))]
        elif kind == "dyadic_small_row":                                 # one row of magnitude < 1 among large ones
            m = int(rng.integers(50, 400))
            v = [float(a) for a in rng.integers(-2 ** 40, 2 ** 40, m)] + [[0.25, -0.5, 0.75][g % 3]]
        elif kind == "ill_conditioned":
            m = int(rng.integers(2, 20))
            big = [float(a) * 1e16 for a in rng.integers(1, 9, m)]
            v = big + [-b for b in big] + fin(n)
        elif kind == "normal":
            v = [float(x) for x in rng.normal(0, 1e6, int(rng.integers(20, 120)))]
        else:
            v = [None] * n
        if kind.startswith("dyadic"):
            assert isinstance(f64_sum(v), float), "a dyadic group must have an order-independent sum"
        if rng.random() < 0.3 and kind != "all_null":
            v = v + [None]
        out.append((kind, v))
    return out


def float_minmax_groups(rng, width, ngroups=600):
    """edge groups of f64 / f32 MIN / MAX: ±0.0 ties, ±NaN, ±inf, the extreme finite values, subnormals"""
    mx = DBL_MAX if width == 64 else F32_MAX
    tiny = DBL_MIN if width == 64 else float(np.finfo(np.float32).tiny)
    sub = SUBNORMAL_MIN if width == 64 else float(np.float32(1e-45))
    kinds = ["zeros", "neg_zero", "pos_nan", "neg_nan", "both_nan", "pinf", "ninf", "extremes", "subnormal", "random", "all_null"]
    out = []
    for g in range(ngroups):
        kind = kinds[g % len(kinds)]
        fin = [float(x) for x in rng.normal(0, 1e3, int(rng.integers(1, 5)))]
        v = {"zeros": [0.0, -0.0, 0.0, -0.0], "neg_zero": [-0.0, -0.0], "pos_nan": fin + [math.nan], "neg_nan": fin + [NEG_NAN],
             "both_nan": fin + [math.nan, NEG_NAN], "pinf": fin + [math.inf], "ninf": fin + [-math.inf],
             "extremes": [-mx, mx, tiny, -tiny], "subnormal": [sub, -sub, sub * 3, 0.0], "random": fin, "all_null": [None, None]}[kind]
        if width == 32:
            v = [None if x is None else to_f32(x) for x in v]
        v = [v[i] for i in rng.permutation(len(v))]
        if rng.random() < 0.3 and kind != "all_null":
            v = v + [None]
        out.append((kind, v))
    return out


def decimal_groups(rng, ngroups=400):
    """edge groups of decimal128: values near ±(10^38 - 1), sums that wrap past ±2^127, 32-bit pieces of all ones (carries
    between the pieces of the wide kernel), equal high words whose low words straddle 2^63 (a signed / unsigned compare),
    negative sums (AVG rounds toward -inf), and a small-precision column for the wide kernel's scaled AVG"""
    kinds = ["near_max", "wrap_pos", "wrap_neg", "carry_pieces", "straddle", "negative", "small", "all_null"]
    out = []
    for g in range(ngroups):
        kind = kinds[g % len(kinds)]
        n = int(rng.integers(2, 8))
        if kind == "near_max":
            v = [int(s) * (BIG - int(d)) for s, d in zip(rng.choice([-1, 1], n), rng.integers(0, 1000, n))]
        elif kind == "wrap_pos":
            v = [BIG - int(d) for d in rng.integers(0, 10 ** 6, n + 2)]              # > 2^127 after two rows
        elif kind == "wrap_neg":
            v = [-BIG + int(d) for d in rng.integers(0, 10 ** 6, n + 2)]
        elif kind == "carry_pieces":
            hi = int(rng.integers(0, 1 << 40))
            v = [(hi << 64) | 0xFFFFFFFFFFFFFFFF, (hi << 64) | 0x00000000FFFFFFFF, 0xFFFFFFFF00000000, 1, (1 << 64) - 1] * 2
        elif kind == "straddle":
            hi = int(rng.integers(-(1 << 40), 1 << 40))
            v = [(hi << 64) + lo for lo in ((1 << 63) - 1, 1 << 63, (1 << 63) + 1, 0, (1 << 64) - 1)]
        elif kind == "negative":
            v = [-int(x) for x in rng.integers(1, 10 ** 18, n)] + [-7]
        elif kind == "small":
            v = [int(x) for x in rng.integers(-10 ** 15, 10 ** 15, n)]
        else:
            v = [None] * n
        if rng.random() < 0.3 and kind != "all_null":
            v = v + [None]
        rng.shuffle(v)
        out.append((kind, v))
    return out


def int_groups(rng, ngroups=400):
    """edge groups of int64: SUMs that wrap several times, INT64_MIN / INT64_MAX only, values above 2^53 whose exact sum
    exceeds 2^63 (AVG through f64)"""
    kinds = ["wrap_many", "extremes_only", "min_only", "max_only", "big_avg", "random", "all_null"]
    out = []
    for g in range(ngroups):
        kind = kinds[g % len(kinds)]
        n = int(rng.integers(2, 8))
        if kind == "wrap_many":
            v = [INT64_MAX - int(d) for d in rng.integers(0, 1000, 6 + n)] + [INT64_MIN] * 2
        elif kind == "extremes_only":
            v = [INT64_MIN, INT64_MAX] * n
        elif kind == "min_only":
            v = [INT64_MIN] * n
        elif kind == "max_only":
            v = [INT64_MAX] * n
        elif kind == "big_avg":
            v = [int(x) for x in rng.integers((1 << 62) + 1, INT64_MAX, n + 2)]       # > 2^53, exact sum > 2^63
        elif kind == "random":
            v = [int(x) for x in rng.integers(-2 ** 40, 2 ** 40, n)]
        else:
            v = [None] * n
        if rng.random() < 0.3 and kind != "all_null":
            v = v + [None]
        rng.shuffle(v)
        out.append((kind, v))
    return out


def narrow_int_values(rng, n):
    """int8 / int16 / int32 columns at their type limits"""
    cols = {}
    for name, bits in (("i8", 8), ("i16", 16), ("i32", 32)):
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        cols[name] = [int(v) for v in rng.choice([lo, hi, lo + 1, hi - 1, 0, -1], n)]
    return cols


# ---- tables --------------------------------------------------------------------------------------------------------------
@dataclass
class Table:
    batches: list            # pa.RecordBatch, the first one decides the dense key range
    keys: list               # per row: the key (int or None)
    cols: dict               # name -> per-row values (None = NULL)
    types: dict              # name -> blaze type
    kinds: dict              # key -> the group's edge kind

    @property
    def schema(self):
        return self.batches[0].schema


def _arrow_column(vals, dt):
    if dt.is_decimal:
        # unscaled 128-bit two's complement words: values up to 10^38 - 1 at any scale
        data = b"".join((0 if v is None else v).to_bytes(16, "little", signed=True) for v in vals)
        valid = np.array([v is not None for v in vals])
        bits = np.packbits(valid.astype(np.uint8), bitorder="little").tobytes()
        return pa.Array.from_buffers(T.to_arrow_type(dt), len(vals), [pa.py_buffer(bits), pa.py_buffer(data)], null_count=int((~valid).sum()))
    return pa.array(vals, type=T.to_arrow_type(dt))


def table(rng, groups, types, *, far_frac=0.06, nbatches=3, key_base=0):
    """lay the groups out as rows.  Most groups take dense keys key_base, key_base + 1, ...; the first batch holds only
    their rows, so the dense key range is theirs.  A few groups take keys far outside that range and one group the NULL
    key: their rows come in the later batches (the hashed fall-back next to a dense table).  Rows are shuffled.
    groups: [(kind, {column: [values]})] with equally long value lists per group"""
    nfar = max(1, int(len(groups) * far_frac))
    gkeys = [key_base + i for i in range(len(groups) - nfar - 1)] + [10 ** 12 + 7919 * i for i in range(nfar)] + [None]
    perm = rng.permutation(len(groups))
    dense_rows, late_rows = [], []
    kinds = {}
    for gi, key in zip(perm, gkeys):
        kind, vals = groups[gi]
        kinds[key] = kind
        m = len(next(iter(vals.values())))
        rows = [(key, {c: vals[c][j] for c in vals}) for j in range(m)]
        (late_rows if key is None or key >= 10 ** 12 else dense_rows).extend(rows)
    dense_rows = [dense_rows[i] for i in rng.permutation(len(dense_rows))]
    n1 = len(dense_rows) // nbatches
    tail = dense_rows[n1:] + late_rows
    rows = dense_rows[:n1] + [tail[i] for i in rng.permutation(len(tail))]
    keys = [r[0] for r in rows]
    cols = {c: [r[1][c] for r in rows] for c in types}
    arrays = [pa.array(keys, pa.int64())] + [_arrow_column(cols[c], types[c]) for c in types]
    rb = pa.RecordBatch.from_arrays(arrays, names=["k"] + list(types))
    step = max(1, (len(rows) - n1 + nbatches - 2) // max(1, nbatches - 1))
    batches = [rb.slice(0, n1)] + [rb.slice(i, min(step, len(rows) - i)) for i in range(n1, len(rows), step)]
    return Table(batches, keys, cols, dict(types), kinds)


def _one_column(groups, name):
    return [(kind, {name: v}) for kind, v in groups]


def family_f64_sum(seed, ngroups=600):
    rng = np.random.default_rng(seed)
    return table(rng, _one_column(f64_sum_groups(rng, ngroups), "x"), {"x": T.float64})


def family_float_minmax(seed, width, ngroups=600):
    rng = np.random.default_rng(seed)
    return table(rng, _one_column(float_minmax_groups(rng, width, ngroups), "x"), {"x": T.float64 if width == 64 else T.float32})


def family_decimal(seed, ngroups=400):
    """columns d0 (decimal(38,0)), d10 (decimal(38,10)), d2 (decimal(38,2), the AVG cast to (38,6) overflows near 10^38)
    and s2 (decimal(20,2), values that fit its precision)"""
    rng = np.random.default_rng(seed)
    groups = []
    for kind, v in decimal_groups(rng, ngroups):
        s2 = [None if x is None else (x if -10 ** 20 < x < 10 ** 20 else (abs(x) % 10 ** 20) * (1 if x > 0 else -1)) for x in v]
        groups.append((kind, {"d0": v, "d10": v, "d2": v, "s2": s2}))
    return table(rng, groups, {"d0": D38_0, "d10": D38_10, "d2": D38_2, "s2": D20_2})


def family_int(seed, ngroups=400):
    rng = np.random.default_rng(seed)
    groups = []
    for kind, v in int_groups(rng, ngroups):
        nar = narrow_int_values(rng, len(v))
        groups.append((kind, {"i": v, **{c: [None if x is None else y for x, y in zip(v, nar[c])] for c in nar}}))
    return table(rng, groups, {"i": T.int64, "i8": T.int8, "i16": T.int16, "i32": T.int32})


def family_extreme_keys(seed, ngroups=300):
    """int64 keys at and next to INT64_MIN in the first batch (the dense base is clamped), the other end of the range in
    later batches (hashed slots), NULL keys beside key 0; dyadic f64 and int64 values"""
    rng = np.random.default_rng(seed)
    keys, xs, vs = [], [], []
    low = [INT64_MIN + i for i in range(ngroups)]
    high = [INT64_MAX - i for i in range(ngroups // 4)] + [0, None]
    first, later = [], []
    for k in low:
        for _ in range(int(rng.integers(1, 5))):
            first.append(k)
    for k in high + low[: ngroups // 4]:
        for _ in range(int(rng.integers(1, 5))):
            later.append(k)
    rng.shuffle(first); rng.shuffle(later)
    keys = first + later
    xs = [float(a) / 4 for a in rng.integers(-2 ** 40, 2 ** 40, len(keys))]
    vs = [int(a) for a in rng.integers(INT64_MIN, INT64_MAX, len(keys), dtype=np.int64)]
    types = {"x": T.float64, "i": T.int64}
    rb = pa.RecordBatch.from_arrays([pa.array(keys, pa.int64()), pa.array(xs, pa.float64()), pa.array(vs, pa.int64())], names=["k", "x", "i"])
    n1 = len(first)
    return Table([rb.slice(0, n1), rb.slice(n1)], keys, {"x": xs, "i": vs}, types, {k: "extreme_key" for k in keys})


# ---- the aggregate shapes the tests run over the families -------------------------------------------------------------
class Shape:
    def __init__(self, family, specs, fast):
        self.family, self.specs, self.fast = family, specs, fast     # fast: the default conf takes a specialised kernel


FAMILIES = {
    "f64": lambda: family_f64_sum(101),
    "f64mm": lambda: family_float_minmax(102, 64),
    "f32mm": lambda: family_float_minmax(103, 32),
    "dec": lambda: family_decimal(104),
    "int": lambda: family_int(105),
    "keys": lambda: family_extreme_keys(106),
}
_tables = {}


def family(name):
    if name not in _tables:
        _tables[name] = FAMILIES[name]()
    return _tables[name]


SHAPES = {
    "f64 sum avg count":   Shape("f64", [("s", E.AGG_SUM, "x", T.float64), ("a", E.AGG_AVG, "x", T.float64), ("c", E.AGG_COUNT, "x", T.int64)], True),
    "f64 min max":         Shape("f64mm", [("mn", E.AGG_MIN, "x", T.float64), ("mx", E.AGG_MAX, "x", T.float64)], True),
    "f32 min max":         Shape("f32mm", [("mn", E.AGG_MIN, "x", T.float32), ("mx", E.AGG_MAX, "x", T.float32)], False),
    "dec38_0 sum count":   Shape("dec", [("s", E.AGG_SUM, "d0", D38_0), ("c", E.AGG_COUNT, "d0", T.int64)], True),
    "dec38_10 sum":        Shape("dec", [("s", E.AGG_SUM, "d10", D38_10)], True),
    "dec20_2 avg scaled":  Shape("dec", [("a", E.AGG_AVG, "s2", T.decimal128(24, 6))], True),
    "dec avg cast min max": Shape("dec", [("a", E.AGG_AVG, "d2", T.decimal128(38, 6)), ("mn", E.AGG_MIN, "d0", D38_0), ("mx", E.AGG_MAX, "d0", D38_0)], False),
    "int sum count":       Shape("int", [("s", E.AGG_SUM, "i", T.int64), ("c", E.AGG_COUNT, "i", T.int64)], True),
    "int min max":         Shape("int", [("mn", E.AGG_MIN, "i", T.int64), ("mx", E.AGG_MAX, "i", T.int64)], True),
    "int avg":             Shape("int", [("a", E.AGG_AVG, "i", T.float64), ("c", E.AGG_COUNT, "i", T.int64)], True),
    "narrow sums":         Shape("int", [("s8", E.AGG_SUM, "i8", T.int64), ("s32", E.AGG_SUM, "i32", T.int64)], True),
    "narrow min max avg":  Shape("int", [("mn", E.AGG_MIN, "i8", T.int8), ("mx", E.AGG_MAX, "i16", T.int16), ("a", E.AGG_AVG, "i32", T.float64)], False),
    "keys f64 sum":        Shape("keys", [("s", E.AGG_SUM, "x", T.float64), ("c", E.AGG_COUNT, "x", T.int64)], True),
    "keys int sum":        Shape("keys", [("s", E.AGG_SUM, "i", T.int64), ("n", E.AGG_COUNT, None, T.int64)], True),
}
