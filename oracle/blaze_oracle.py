"""CPU ORACLE — TEST INFRASTRUCTURE ONLY.  Nothing under `blaze_b200/` may import this module.

A numpy restatement of the reference's Filter / Project / HashAgg semantics
(kwai/blaze = Apache Auron @ d1eaef148a58), used by `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s cpu_baseline leg as the checker for the CUDA path.  Each function cites the
reference file:line it follows (paths relative to the reference's native-engine/).

PARITY STATUS
  * HashAgg (Sum/Count/Avg/Min/Max, Partial/PartialMerge/Final, frozen-row bytes, varint):
    pinned by the reference's own KAT `test_agg` (datafusion-ext-plans/src/agg_exec.rs:493-681)
    and the fuzz model (:714-843) — see tests/test_oracle_golden.py.
  * murmur3 / pmod partition ids: pinned by datafusion-ext-commons/src/hash/mur.rs:94-103 and
    spark_hash.rs:377-456.
  * CheckOverflow / MakeDecimal / UnscaledValue: pinned by the KATs in
    datafusion-ext-functions/src/spark_check_overflow.rs:134-158 (and siblings).
  * Filter / Project / expression evaluation (BinaryExpr, Kleene And/Or, comparisons, Case,
    InList, casts): **parity unpinned** — the reference has no native golden for them and the
    arithmetic lives in un-vendored forks (datafusion 49.0.0 @ 9034aeffb, arrow-rs 55.2.0 @
    5de02520c; Cargo.toml:111-137).  Restated from the published upstream semantics; every
    such assumption is marked `ASSUMPTION(df49/arrow55)` below, and cross-checked
    differentially against pyarrow.compute in tests/test_oracle_vs_pyarrow.py.
"""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from blaze_b200 import exprs as E
from blaze_b200 import types as T
from blaze_b200.types import DataType, Field, Schema

np.seterr(over="ignore", invalid="ignore", divide="ignore")

I128_MASK = (1 << 128) - 1


def wrap_i128(v: int) -> int:
    v &= I128_MASK
    return v - (1 << 128) if v >> 127 else v


def wrap_i64(v: int) -> int:
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


_NP = {T.BOOL: np.bool_, T.INT8: np.int8, T.INT16: np.int16, T.INT32: np.int32, T.INT64: np.int64,
       T.FLOAT32: np.float32, T.FLOAT64: np.float64, T.DATE32: np.int32, T.TIMESTAMP_US: np.int64,
       T.DECIMAL128: object, T.BINARY: object, T.NULLTYPE: np.int8}


class OracleError(Exception):
    """an error the reference would raise as DataFusionError / ArrowError"""


@dataclass
class Col:
    dtype: DataType
    values: np.ndarray
    valid: np.ndarray          # bool per row
    is_scalar: bool = False    # DataFusion ColumnarValue::Scalar

    def __len__(self):
        return len(self.values)

    @staticmethod
    def nulls(dtype: DataType, n: int) -> "Col":
        return Col(dtype, _zeros(dtype, n), np.zeros(n, bool))

    def take(self, idx) -> "Col":
        return Col(self.dtype, self.values[idx], self.valid[idx])

    def broadcast(self, n: int) -> "Col":
        if not self.is_scalar:
            assert len(self) == n
            return self
        return Col(self.dtype, np.repeat(self.values, n), np.repeat(self.valid, n))


def _zeros(dtype: DataType, n: int) -> np.ndarray:
    if dtype.id == T.DECIMAL128:
        a = np.empty(n, object); a[:] = 0
        return a
    if dtype.id == T.BINARY:
        a = np.empty(n, object); a[:] = b""
        return a
    return np.zeros(n, _NP[dtype.id])


@dataclass
class Batch:
    schema: Schema
    cols: List[Col]
    num_rows: int

    @staticmethod
    def empty(schema: Schema) -> "Batch":
        return Batch(schema, [Col.nulls(f.dtype, 0) for f in schema], 0)

    def take(self, idx) -> "Batch":
        idx = np.asarray(idx)
        n = int(idx.sum()) if idx.dtype == bool else len(idx)
        return Batch(self.schema, [c.take(idx) for c in self.cols], n)


# ---- pyarrow bridges ---------------------------------------------------------------------------

def col_from_arrow(arr) -> Col:
    import pyarrow as pa
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    dt = T.from_arrow_type(arr.type)
    n = len(arr)
    valid = np.ones(n, bool) if arr.null_count == 0 else np.array(arr.is_valid().to_pylist(), bool)
    if dt.id == T.DECIMAL128:
        # the unscaled 128-bit words themselves: a Decimal through the default 28-digit context would round them
        words = np.frombuffer(arr.buffers()[1], dtype="<u8", count=2 * (arr.offset + n))[2 * arr.offset:] if n else []
        vals = np.empty(n, object)
        for i in range(n):
            vals[i] = wrap_i128(int(words[2 * i]) | int(words[2 * i + 1]) << 64) if valid[i] else 0
    elif dt.id == T.BINARY:
        vals = np.empty(n, object)
        for i, v in enumerate(arr.to_pylist()):
            vals[i] = b"" if v is None else v
    elif dt.id == T.BOOL:
        vals = np.array([bool(v) for v in arr.fill_null(False).to_pylist()], bool) if n else np.zeros(0, bool)
    elif dt.id == T.NULLTYPE:
        vals = np.zeros(n, np.int8); valid = np.zeros(n, bool)
    else:
        npdt = _NP[dt.id]
        if dt.id in (T.DATE32, T.TIMESTAMP_US):
            arr = arr.cast(pa.int32() if dt.id == T.DATE32 else pa.int64())
        zero = pa.scalar(0, arr.type)
        vals = np.asarray(arr.fill_null(zero).to_numpy(zero_copy_only=False), dtype=npdt).copy()
    return Col(dt, vals, valid)


def col_to_arrow(c: Col):
    import decimal
    import pyarrow as pa
    at = T.to_arrow_type(c.dtype)
    mask = ~c.valid
    if c.dtype.id == T.DECIMAL128:
        # raw 128-bit little-endian words, no precision validation: MakeDecimal / Decimal128Array::from(..)
        # .with_precision_and_scale keep out-of-precision unscaled values as they are (spark_make_decimal.rs:24-58)
        data = b"".join((int(v) if ok else 0).to_bytes(16, "little", signed=True) for v, ok in zip(c.values, c.valid))
        bits = np.packbits(np.asarray(c.valid, dtype=np.uint8), bitorder="little").tobytes()
        return pa.Array.from_buffers(at, len(c), [pa.py_buffer(bits), pa.py_buffer(data)], null_count=int(mask.sum()))
    if c.dtype.id == T.BINARY:
        return pa.array([None if not ok else bytes(v) for v, ok in zip(c.values, c.valid)], type=at)
    if c.dtype.id == T.NULLTYPE:
        return pa.nulls(len(c))
    if c.dtype.id == T.DATE32:
        return pa.array(c.values.astype(np.int32), mask=mask, type=pa.int32()).cast(at)
    if c.dtype.id == T.TIMESTAMP_US:
        return pa.array(c.values.astype(np.int64), mask=mask, type=pa.int64()).cast(at)
    return pa.array(c.values, mask=mask, type=at)


def batch_from_arrow(rb) -> Batch:
    schema = T.from_arrow_schema(rb.schema)
    return Batch(schema, [col_from_arrow(rb.column(i)) for i in range(rb.num_columns)], rb.num_rows)


def batch_to_arrow(b: Batch):
    import pyarrow as pa
    return pa.RecordBatch.from_arrays([col_to_arrow(c) for c in b.cols], schema=T.to_arrow_schema(b.schema))


# =================================================================================================
# Expression evaluation (DataFusion PhysicalExpr::evaluate; un-vendored — ASSUMPTION(df49/arrow55))
# =================================================================================================

def _int_info(dt: DataType):
    return np.iinfo(_NP[dt.id])


def _scalar(dtype: DataType, value) -> Col:
    vals = _zeros(dtype, 1)
    ok = value is not None
    if ok:
        vals[0] = value
    return Col(dtype, vals, np.array([ok]), is_scalar=True)


def evaluate(expr: E.Expr, batch: Batch) -> Col:
    """PhysicalExpr::evaluate.  Result is_scalar iff every leaf is a literal."""
    n = batch.num_rows
    s = batch.schema
    if isinstance(expr, E.Column):
        return batch.cols[s.index_of(expr.name)]
    if isinstance(expr, E.BoundReference):
        return batch.cols[expr.index]
    if isinstance(expr, E.Literal):
        return _scalar(expr.dtype, expr.value)
    if isinstance(expr, E.BinaryExpr):
        l, r = evaluate(expr.left, batch), evaluate(expr.right, batch)
        return _binary(expr.op, l, r, n)
    if isinstance(expr, (E.SCAnd, E.SCOr)):
        # fork-only SCAndExpr/SCOrExpr (from_proto.rs:1010-1019): evaluates the right side only
        # under the left's selection; for pure expressions the truth table is Kleene And/Or.
        l, r = evaluate(expr.left, batch), evaluate(expr.right, batch)
        return _binary("And" if isinstance(expr, E.SCAnd) else "Or", l, r, n)
    if isinstance(expr, E.IsNull):
        c = evaluate(expr.expr, batch)
        return Col(T.bool_, ~c.valid, np.ones(len(c), bool), c.is_scalar)
    if isinstance(expr, E.IsNotNull):
        c = evaluate(expr.expr, batch)
        return Col(T.bool_, c.valid.copy(), np.ones(len(c), bool), c.is_scalar)
    if isinstance(expr, E.Not):
        c = evaluate(expr.expr, batch)
        return Col(T.bool_, ~c.values.astype(bool), c.valid, c.is_scalar)
    if isinstance(expr, E.Negative):
        c = evaluate(expr.expr, batch)
        if c.dtype.is_decimal:
            v = np.array([wrap_i128(-int(x)) for x in c.values], object) if len(c) else c.values
            return Col(c.dtype, v, c.valid, c.is_scalar)
        return Col(c.dtype, (-c.values).astype(c.values.dtype), c.valid, c.is_scalar)   # neg_wrapping
    if isinstance(expr, (E.Cast, E.TryCast)):
        c = evaluate(expr.expr, batch)
        out = cast(c, expr.dtype)
        out.is_scalar = c.is_scalar
        return out
    if isinstance(expr, E.Case):
        return _case(expr, batch)
    if isinstance(expr, E.InList):
        return _in_list(expr, batch)
    if isinstance(expr, E.ScalarFunction):
        return _scalar_function(expr, batch)
    raise OracleError(f"unsupported expression {expr!r}")


def _common_len(l: Col, r: Col, n: int) -> Tuple[Col, Col, bool]:
    if l.is_scalar and r.is_scalar:
        return l, r, True
    return l.broadcast(n), r.broadcast(n), False


def _total_order_key(a: np.ndarray) -> np.ndarray:
    """IEEE-754 totalOrder as a signed-integer key: arrow-rs compares floats with `total_cmp`
    (arrow-array ArrowNativeTypeOp::is_lt / is_eq for f32/f64).  ASSUMPTION(df49/arrow55)."""
    if a.dtype == np.float64:
        b = a.view(np.int64)
        return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))
    b = a.astype(np.float32).view(np.int32)
    return b ^ ((b >> 31) & np.int32(0x7FFFFFFF))


def _cmp_arrays(op: str, a, b):
    return {"Eq": a == b, "NotEq": a != b, "Lt": a < b, "LtEq": a <= b, "Gt": a > b, "GtEq": a >= b}[op]


def _binary(op: str, l: Col, r: Col, n: int) -> Col:
    l, r, sc = _common_len(l, r, n)
    if op in ("And", "Or"):
        # Kleene three-valued logic (arrow and_kleene / or_kleene)
        lv, rv = l.values.astype(bool), r.values.astype(bool)
        if op == "And":
            lf, rf = l.valid & ~lv, r.valid & ~rv
            valid = (l.valid & r.valid) | lf | rf
            vals = lv & rv & l.valid & r.valid
        else:
            lt, rt = l.valid & lv, r.valid & rv
            valid = (l.valid & r.valid) | lt | rt
            vals = lt | rt
        return Col(T.bool_, vals, valid, sc)
    valid = l.valid & r.valid
    if op in E.COMPARISONS:
        if l.dtype.is_decimal or r.dtype.is_decimal:
            if l.dtype.scale != r.dtype.scale or not (l.dtype.is_decimal and r.dtype.is_decimal):
                raise OracleError(f"compare {l.dtype} with {r.dtype}: arrow cmp requires equal types")
            vals = np.array([_cmp_arrays(op, int(a), int(b)) for a, b in zip(l.values, r.values)], bool) \
                if len(l) else np.zeros(0, bool)
        elif l.dtype != r.dtype:
            raise OracleError(f"compare {l.dtype} with {r.dtype}: arrow cmp requires equal types")
        elif l.dtype.is_float:
            vals = _cmp_arrays(op, _total_order_key(l.values), _total_order_key(r.values))
        else:
            vals = _cmp_arrays(op, l.values, r.values)
        return Col(T.bool_, np.asarray(vals, bool), valid, sc)
    if op in E.BITWISE:
        if l.dtype != r.dtype or not l.dtype.is_integer:
            raise OracleError(f"bitwise {op} on {l.dtype},{r.dtype}")
        f = {"BitwiseAnd": np.bitwise_and, "BitwiseOr": np.bitwise_or, "BitwiseXor": np.bitwise_xor}[op]
        return Col(l.dtype, f(l.values, r.values), valid, sc)
    # arithmetic
    if l.dtype.is_decimal and r.dtype.is_decimal:
        return _decimal_arith(op, l, r, valid, sc)
    if l.dtype != r.dtype:
        raise OracleError(f"{op} on {l.dtype},{r.dtype}: arrow arithmetic requires equal types")
    dt = l.dtype
    a, b = l.values, r.values
    if dt.is_float:
        if op == "Plus": v = a + b
        elif op == "Minus": v = a - b
        elif op == "Multiply": v = a * b
        elif op == "Divide": v = a / b                       # div_wrapping: IEEE, never errors
        else: v = np.fmod(a, b)                              # mod_wrapping: Rust `%` == C fmod
        return Col(dt, v.astype(a.dtype), valid, sc)
    if not dt.is_integer:
        raise OracleError(f"{op} on {dt}")
    if op == "Plus": v = a + b                               # add_wrapping (fail_on_overflow=false)
    elif op == "Minus": v = a - b
    elif op == "Multiply": v = a * b
    else:
        # integer Divide/Modulo = div_checked / mod_checked on valid slots: error on /0 and MIN/-1
        bz = (b == 0) & valid
        if bz.any():
            raise OracleError("Arrow error: Divide by zero error")
        info = _int_info(dt)
        ov = (a == info.min) & (b == -1) & valid
        if ov.any():
            raise OracleError("Arrow error: Arithmetic overflow")
        bb = np.where(valid, b, 1)
        if op == "Divide":
            q = np.abs(a.astype(object)) // np.abs(bb.astype(object))   # truncating division
            q = np.where((a < 0) != (bb < 0), -q, q)
            v = q.astype(a.dtype) if len(a) else a
        else:
            v = np.fmod(a, bb)                                           # sign follows dividend
    return Col(dt, v.astype(a.dtype), valid, sc)


def _decimal_arith(op: str, l: Col, r: Col, valid, sc) -> Col:
    """arrow-arith decimal_op for Add/Sub: rescale both sides to max(scale), checked i128
    arithmetic (error on i128 overflow).  ASSUMPTION(df49/arrow55)."""
    out_t = E.decimal_result_type(op, l.dtype, r.dtype)
    lm, rm = 10 ** (out_t.scale - l.dtype.scale), 10 ** (out_t.scale - r.dtype.scale)
    vals = np.empty(len(l), object)
    for i in range(len(l)):
        if not valid[i]:
            vals[i] = 0
            continue
        a, b = int(l.values[i]) * lm, int(r.values[i]) * rm
        v = a + b if op == "Plus" else a - b
        if not (-(1 << 127) <= v < (1 << 127)):
            raise OracleError("Arrow error: Arithmetic overflow")
        vals[i] = v
    return Col(out_t, vals, valid, sc)


def _case(expr: E.Case, batch: Batch) -> Col:
    n = batch.num_rows
    out_t = expr.data_type(batch.schema)
    vals, valid = _zeros(out_t, n), np.zeros(n, bool)
    remaining = np.ones(n, bool)
    base = evaluate(expr.expr, batch).broadcast(n) if expr.expr is not None else None
    for w, t in expr.when_then:
        wc = evaluate(w, batch).broadcast(n)
        if base is not None:
            wc = _binary("Eq", base, wc, n)
        hit = remaining & wc.valid & wc.values.astype(bool)
        tc = evaluate(t, batch).broadcast(n)
        if tc.dtype.id != T.NULLTYPE:
            vals[hit] = tc.values[hit]
            valid[hit] = tc.valid[hit]
        remaining &= ~hit
    if expr.else_expr is not None:
        ec = evaluate(expr.else_expr, batch).broadcast(n)
        if ec.dtype.id != T.NULLTYPE:
            vals[remaining] = ec.values[remaining]
            valid[remaining] = ec.valid[remaining]
    return Col(out_t, vals, valid)


def _in_list(expr: E.InList, batch: Batch) -> Col:
    n = batch.num_rows
    x = evaluate(expr.expr, batch).broadcast(n)
    found = np.zeros(n, bool)
    any_null_item = np.zeros(n, bool)
    for item in expr.list:
        ic = evaluate(item, batch).broadcast(n)
        if ic.dtype != x.dtype:                       # from_proto.rs:888-895 wraps a TryCast
            ic = cast(ic, x.dtype)
        eq = _binary("Eq", x, ic, n)
        found |= eq.valid & eq.values
        any_null_item |= ~ic.valid
    valid = x.valid & (found | ~any_null_item)
    vals = found != expr.negated
    return Col(T.bool_, vals, valid)


def change_precision_round_half_up(v: int, precision: int, scale: int, to_p: int, to_s: int) -> Optional[int]:
    """datafusion-ext-functions/src/spark_check_overflow.rs:84-124"""
    if to_p == precision and to_s == scale:
        return v
    if to_s < scale:
        p10 = 10 ** (scale - to_s)
        q = abs(v) // p10
        rem = abs(v) - q * p10
        v = -q if v < 0 else q                       # `/` and `%` round toward zero
        if rem * 2 >= p10:
            v += -1 if (v < 0 or (v == 0 and _neg_zero_helper)) else 1 if False else 0  # replaced below
    elif to_s > scale:
        v = wrap_i128(v * 10 ** (to_s - scale))
    p = 10 ** min(to_p, 38)
    if v <= -p or v >= p:
        return None
    return v


_neg_zero_helper = False


def _change_precision(v: int, precision: int, scale: int, to_p: int, to_s: int) -> Optional[int]:
    """datafusion-ext-functions/src/spark_check_overflow.rs:84-124 (the version actually used)"""
    if to_p == precision and to_s == scale:
        return v
    if to_s < scale:
        p10 = 10 ** (scale - to_s)
        neg = v < 0
        q, rem = divmod(abs(v), p10)
        v = -q if neg else q                         # Rust `/` and `%` round toward zero
        dropped = -rem if neg else rem
        if wrap_i128(abs(dropped) * 2) >= p10:         # release build: the i128 product wraps (no rounding for |dropped| >= 2^126)
            v += -1 if dropped < 0 else 1
    elif to_s > scale:
        v = wrap_i128(v * 10 ** (to_s - scale))      # release build: wrapping multiply
    p = 10 ** min(to_p, 38)
    if v <= -p or v >= p:
        return None
    return v


change_precision_round_half_up = _change_precision  # noqa: F811  (public name)


def _scalar_function(expr: E.ScalarFunction, batch: Batch) -> Col:
    n = batch.num_rows
    name = expr.name
    if name == "Placeholder":
        raise OracleError("placeholder() should never be called")
    args = [evaluate(a, batch) for a in expr.args]
    sc = all(a.is_scalar for a in args)
    if name == "UnscaledValue":
        # spark_unscaled_value.rs:24-42: Decimal128 -> Int64 by `as i64` (low 64 bits)
        a = args[0]
        vals = np.array([wrap_i64(int(v)) for v in a.values], np.int64) if len(a) else np.zeros(0, np.int64)
        return Col(T.int64, vals, a.valid.copy(), sc)
    if name == "MakeDecimal":
        # spark_make_decimal.rs:24-58: Int64 -> Decimal128(p,s), no range check
        a = args[0]
        p, s = int(args[1].values[0]), int(args[2].values[0])
        vals = np.array([int(v) for v in a.values], object) if len(a) else np.zeros(0, object)
        return Col(T.decimal128(p, s), vals, a.valid.copy(), sc)
    if name == "CheckOverflow":
        a = args[0]
        p, s = int(args[1].values[0]), int(args[2].values[0])
        vals, valid = np.empty(len(a), object), a.valid.copy()
        for i in range(len(a)):
            r = change_precision_round_half_up(int(a.values[i]), a.dtype.precision, a.dtype.scale, p, s) if valid[i] else None
            if r is None:
                vals[i], valid[i] = 0, False
            else:
                vals[i] = r
        return Col(T.decimal128(p, s), vals, valid, sc)
    if name == "NullIfZero":
        # spark_null_if.rs: value == 0 -> NULL (used to avoid divide-by-zero errors)
        a = args[0]
        if a.dtype.is_decimal:
            z = np.array([int(v) == 0 for v in a.values], bool) if len(a) else np.zeros(0, bool)
        else:
            z = a.values == 0
        return Col(a.dtype, a.values, a.valid & ~z, sc)
    if name == "NullIf":
        a, b = args[0].broadcast(n) if not sc else args[0], args[1].broadcast(n) if not sc else args[1]
        eq = _binary("Eq", a, b, n)
        return Col(a.dtype, a.values, a.valid & ~(eq.valid & eq.values), sc)
    if name == "NormalizeNanAndZero":
        a = args[0]
        v = a.values.copy()
        v[np.isnan(v)] = np.nan
        v[v == 0] = 0.0
        return Col(a.dtype, v, a.valid.copy(), sc)
    raise OracleError(f"spark ext function not implemented: {name}")


# ---- cast (datafusion-ext-commons/src/arrow/cast.rs:26-225 + arrow-cast defaults) ---------------

def _rust_float_to_int(v: np.ndarray, dt: DataType) -> np.ndarray:
    """Rust `as`: truncate toward zero, saturate, NaN -> 0 (cast.rs:54-95)."""
    info = _int_info(dt)
    f = np.trunc(v.astype(np.float64))
    out = np.zeros(len(v), _NP[dt.id])
    ok = ~np.isnan(f)
    hi = f >= float(info.max)       # float(2^63-1) == 2^63: anything >= saturates
    lo = f <= float(info.min)
    mid = ok & ~hi & ~lo
    out[mid] = f[mid].astype(_NP[dt.id])
    out[ok & hi] = info.max
    out[ok & lo] = info.min
    return out


def cast(c: Col, to: DataType) -> Col:
    frm = c.dtype
    n = len(c)
    if frm == to:
        return Col(to, c.values, c.valid)                                # cast.rs:41
    if to.id == T.NULLTYPE:
        return Col.nulls(to, n)
    if frm.id == T.NULLTYPE:
        return Col.nulls(to, n)
    valid = c.valid.copy()
    # float -> int: unchecked Rust `as` (cast.rs:54-95)
    if frm.is_float and to.is_integer:
        return Col(to, _rust_float_to_int(c.values, to), valid)
    # everything below is arrow-cast 55.2 with CastOptions::default() (safe=true → NULL on failure)
    # ASSUMPTION(df49/arrow55)
    if frm.is_integer and to.is_integer:
        info = _int_info(to)
        ok = (c.values >= info.min) & (c.values <= info.max)
        return Col(to, np.where(ok, c.values, 0).astype(_NP[to.id]), valid & ok)
    if (frm.is_integer or frm.is_float) and to.is_float:
        return Col(to, c.values.astype(_NP[to.id]), valid)
    if frm.id == T.BOOL and (to.is_integer or to.is_float):
        return Col(to, c.values.astype(_NP[to.id]), valid)
    if (frm.is_integer or frm.is_float) and to.id == T.BOOL:
        return Col(to, c.values != 0, valid)
    if frm.id == T.DATE32 and to.id == T.INT32 or frm.id == T.INT32 and to.id == T.DATE32:
        return Col(to, c.values.astype(np.int32), valid)
    if frm.id == T.TIMESTAMP_US and to.id == T.INT64 or frm.id == T.INT64 and to.id == T.TIMESTAMP_US:
        return Col(to, c.values.astype(np.int64), valid)
    if frm.id == T.TIMESTAMP_US and to.id == T.FLOAT64:                  # cast.rs:97-103
        return Col(to, c.values.astype(np.float64), valid)
    if frm.is_integer and to.is_decimal:
        vals = np.empty(n, object)
        m, lim = 10 ** to.scale if to.scale >= 0 else None, 10 ** to.precision
        for i in range(n):
            v = int(c.values[i]) * m if m is not None else int(c.values[i]) // (10 ** -to.scale)
            if valid[i] and -lim < v < lim and -(1 << 127) <= v < (1 << 127):
                vals[i] = v
            else:
                vals[i], valid[i] = 0, False
        return Col(to, vals, valid)
    if frm.is_decimal and to.is_decimal:
        vals = np.empty(n, object)
        lim = 10 ** to.precision
        for i in range(n):
            v = int(c.values[i])
            if to.scale < frm.scale:
                # round half away from zero (arrow-cast cast_decimal_to_decimal)
                p10 = 10 ** (frm.scale - to.scale)
                q, rem = divmod(abs(v), p10)
                if rem * 2 >= p10:
                    q += 1
                v = -q if v < 0 else q
            else:
                v = v * 10 ** (to.scale - frm.scale)
            if valid[i] and -lim < v < lim and -(1 << 127) <= v < (1 << 127):
                vals[i] = v
            else:
                vals[i], valid[i] = 0, False
        return Col(to, vals, valid)
    if frm.is_decimal and to.is_integer:
        info = _int_info(to)
        vals = np.zeros(n, _NP[to.id])
        p10 = 10 ** frm.scale
        for i in range(n):
            v = int(c.values[i])
            q = abs(v) // p10
            q = -q if v < 0 else q                                       # truncate toward zero
            if valid[i] and info.min <= q <= info.max:
                vals[i] = q
            else:
                valid[i] = False
        return Col(to, vals, valid)
    if frm.is_decimal and to.is_float:
        p10 = float(10 ** frm.scale)
        vals = np.array([float(int(v)) / p10 for v in c.values], np.float64).astype(_NP[to.id]) if n else np.zeros(0, _NP[to.id])
        return Col(to, vals, valid)
    if frm.is_float and to.is_decimal:
        vals = np.empty(n, object)
        lim = 10 ** to.precision
        mul = float(10 ** to.scale)
        for i in range(n):
            f = float(c.values[i]) * mul
            if valid[i] and math.isfinite(f):
                q = Fraction(f)                                          # f64::round: half away from zero, exactly
                r = math.floor(abs(q) + Fraction(1, 2))                  # (floor(|f| + 0.5) in f64 rounds the sum first)
                r = -r if f < 0 else r
                if -lim < r < lim:
                    vals[i] = r
                    continue
            vals[i], valid[i] = 0, False
        return Col(to, vals, valid)
    raise OracleError(f"cast {frm} -> {to} is not on the hot path")


# =================================================================================================
# FilterExec / ProjectExec  (datafusion-ext-plans/src/common/cached_exprs_evaluator.rs)
# =================================================================================================

ALL_RETAINED, ALL_FILTERED = "AllRetained", "AllFiltered"


def evaluate_selection(expr: E.Expr, batch: Batch, selection: np.ndarray) -> Col:
    """DataFusion PhysicalExpr::evaluate_selection: evaluate on the selected rows only, scatter the
    result back with NULL in unselected slots.  ASSUMPTION(df49/arrow55)."""
    sub = batch.take(selection)
    res = evaluate(expr, sub)
    if sub.num_rows == batch.num_rows or res.is_scalar:
        return res
    out = Col.nulls(res.dtype, batch.num_rows)
    out.values[selection] = res.values
    out.valid[selection] = res.valid
    return out


def filter_one_pred(batch: Batch, pred: E.Expr, current):
    """cached_exprs_evaluator.rs:495-524"""
    if isinstance(current, str) and current == ALL_FILTERED:
        return ALL_FILTERED
    if isinstance(current, str):
        ret = evaluate(pred, batch)
    else:
        ret = evaluate_selection(pred, batch, current)
    if ret.dtype.id != T.BOOL:
        raise OracleError("filter predicate must be boolean")
    if ret.is_scalar:
        if ret.valid[0] and bool(ret.values[0]):
            return current                                              # :513
        return ALL_FILTERED                                             # :514-516
    return ret.values.astype(bool) & ret.valid                          # null -> false (:518-520)


def filter_batch(predicates: Sequence[E.Expr], batch: Batch) -> Batch:
    """CachedExprsEvaluator::filter_impl (cached_exprs_evaluator.rs:90-136), CSE cache omitted
    (a pure optimisation: cached values are re-filtered to stay row-aligned, :106-128)."""
    current = ALL_RETAINED
    for p in predicates:
        current = filter_one_pred(batch, p, current)
        if isinstance(current, str) and current == ALL_FILTERED:
            return Batch.empty(batch.schema)
    if isinstance(current, str):
        return batch
    return batch.take(current)


def filter_project_batch(predicates, projections, out_schema: Schema, batch: Batch) -> Batch:
    """CachedExprsEvaluator::filter_project_impl (cached_exprs_evaluator.rs:138-166)"""
    fb = filter_batch(predicates, batch)
    if fb.num_rows == 0:
        return Batch.empty(out_schema)
    cols = []
    for e, f in zip(projections, out_schema):
        c = evaluate(e, fb).broadcast(fb.num_rows)
        if c.dtype != f.dtype:
            c = cast(c, f.dtype)                                        # :154-156
        cols.append(Col(c.dtype, c.values, c.valid))
    return Batch(out_schema, cols, fb.num_rows)


class FilterExec:
    """datafusion-ext-plans/src/filter_exec.rs:44-198"""

    def __init__(self, predicates: Sequence[E.Expr], input_schema: Schema):
        if len(predicates) == 0:
            raise OracleError("Filter requires at least one predicate")             # :58-60
        for p in predicates:
            if p.data_type(input_schema).id != T.BOOL:
                raise OracleError("Filter predicate must return boolean values")    # :61-66
        self.predicates = list(predicates)
        self.schema = input_schema

    def execute(self, batches: Sequence[Batch]) -> List[Batch]:
        out = []
        for b in batches:
            fb = filter_batch(self.predicates, b)
            if fb.num_rows > 0:                 # sender.send drops empty batches (execution_context.rs:713-716)
                out.append(fb)
        return out


class ProjectExec:
    """datafusion-ext-plans/src/project_exec.rs:48-232; `predicates` = the fused child FilterExec's
    predicates (:143-149), empty when the child is not a FilterExec."""

    def __init__(self, exprs: Sequence[Tuple[E.Expr, str]], input_schema: Schema, predicates: Sequence[E.Expr] = ()):
        self.exprs = [e for e, _ in exprs]
        self.predicates = list(predicates)
        self.input_schema = input_schema
        self.schema = Schema(Field(name, e.data_type(input_schema), e.nullable(input_schema)) for e, name in exprs)  # :62-72

    def execute(self, batches: Sequence[Batch]) -> List[Batch]:
        out = []
        for b in batches:
            pb = filter_project_batch(self.predicates, self.exprs, self.schema, b)
            if pb.num_rows > 0:
                out.append(pb)
        return out


# =================================================================================================
# varint + frozen accumulator rows
# =================================================================================================

def write_len(n: int) -> bytes:
    """datafusion-ext-commons/src/io/mod.rs:60-68"""
    out = bytearray()
    n &= (1 << 64) - 1                              # `as usize`
    while n >= 128:
        out.append(128 + n % 128)
        n //= 128
    out.append(n)
    return bytes(out)


def read_len(buf: bytes, pos: int) -> Tuple[int, int]:
    """datafusion-ext-commons/src/io/mod.rs:70-83 -> (value, new_pos)"""
    n, factor = 0, 1
    while True:
        v = buf[pos]; pos += 1
        if v < 128:
            return n + v * factor, pos
        n += (v - 128) * factor
        factor *= 128


_PRIM_FMT = {T.INT8: "<b", T.INT16: "<h", T.INT32: "<i", T.INT64: "<q", T.FLOAT32: "<f", T.FLOAT64: "<d",
             T.DATE32: "<i", T.TIMESTAMP_US: "<q"}


def _prim_to_bytes(dt: DataType, v) -> bytes:
    if dt.id == T.DECIMAL128:
        return (int(v) & I128_MASK).to_bytes(16, "little")
    return struct.pack(_PRIM_FMT[dt.id], v)


def _prim_from_bytes(dt: DataType, buf: bytes, pos: int):
    if dt.id == T.DECIMAL128:
        return wrap_i128(int.from_bytes(buf[pos:pos + 16], "little")), pos + 16
    fmt = _PRIM_FMT[dt.id]
    w = struct.calcsize(fmt)
    return struct.unpack_from(fmt, buf, pos)[0], pos + w


# =================================================================================================
# Aggregates (datafusion-ext-plans/src/agg/*)
# =================================================================================================

class _PrimAcc:
    """AccPrimColumn<T> (agg/acc.rs:243-365) / AccBooleanColumn (:101-241)"""

    def __init__(self, dt: DataType):
        self.dt = dt
        self.values: list = []
        self.valids: List[bool] = []

    def resize(self, n):
        zero = False if self.dt.id == T.BOOL else 0
        while len(self.values) < n:
            self.values.append(zero); self.valids.append(False)
        del self.values[n:]; del self.valids[n:]

    def update_value(self, i, default, fn):             # acc.rs:273-280
        if self.valids[i]:
            self.values[i] = fn(self.values[i])
        else:
            self.values[i] = default
            self.valids[i] = True

    def freeze(self, i) -> bytes:                       # acc.rs:335-346 / :180-190
        if self.dt.id == T.BOOL:
            return bytes([1 + int(self.values[i])]) if self.valids[i] else b"\x00"
        if not self.valids[i]:
            return b"\x00"
        return b"\x01" + _prim_to_bytes(self.dt, self.values[i])

    def unfreeze_push(self, buf, pos):                  # acc.rs:349-365 / :193-207
        b = buf[pos]; pos += 1
        if self.dt.id == T.BOOL:
            self.values.append(b - 1 != 0 if b else False); self.valids.append(b != 0)
            return pos
        if b == 1:
            v, pos = _prim_from_bytes(self.dt, buf, pos)
            self.values.append(v); self.valids.append(True)
        else:
            self.values.append(0); self.valids.append(False)
        return pos

    def to_col(self, idx) -> Col:
        vals = _zeros(self.dt, len(idx))
        valid = np.zeros(len(idx), bool)
        for j, i in enumerate(idx):
            if self.valids[i]:
                vals[j] = self.values[i]; valid[j] = True
        return Col(self.dt, vals, valid)


class _CountAcc:
    """AccCountColumn (agg/count.rs:164-229)"""

    def __init__(self):
        self.values: List[int] = []

    def resize(self, n):
        while len(self.values) < n:
            self.values.append(0)
        del self.values[n:]

    def freeze(self, i) -> bytes:
        return write_len(self.values[i])                # `as usize` varint (count.rs:193-203)

    def unfreeze_push(self, buf, pos):
        v, pos = read_len(buf, pos)
        self.values.append(wrap_i64(v))                 # `as i64` (count.rs:205-211)
        return pos


def _np_scalar(dt: DataType, v):
    if dt.id == T.DECIMAL128:
        return int(v)
    return _NP[dt.id](v)


def _add(dt: DataType, a, b):
    """`v + partial_value` (agg/sum.rs:105): wrapping for integers/i128 in release builds
    (Cargo.toml:43-45 overflow-checks=false), IEEE for floats."""
    if dt.id == T.DECIMAL128:
        return wrap_i128(int(a) + int(b))
    if dt.is_integer or dt.id in (T.DATE32, T.TIMESTAMP_US):
        bits = dt.bit_width
        v = (int(a) + int(b)) & ((1 << bits) - 1)
        return _NP[dt.id](v - (1 << bits) if v >> (bits - 1) else v)
    return _NP[dt.id](a) + _NP[dt.id](b)


def _partial_cmp(dt: DataType, a, b):
    """Rust PartialOrd::partial_cmp -> 'Less'|'Equal'|'Greater'|None (None when a float is NaN)"""
    if dt.is_float and (a != a or b != b):
        return None
    return "Less" if a < b else ("Greater" if a > b else "Equal")


class Agg:
    """one aggregate function instance = what `create_agg` returns (agg/agg.rs:171-205)"""

    def __init__(self, fexpr: E.AggFunctionExpr, input_schema: Schema):
        f, ch, rt = fexpr.function, list(fexpr.children), fexpr.return_type
        self.function = f
        if f == E.AGG_COUNT:
            self.data_type = T.int64
            self.exprs = [c for c in ch if c.nullable(input_schema)]          # agg.rs:178-189
            self.nullable = False
        elif f in (E.AGG_SUM, E.AGG_AVG):
            self.data_type = rt
            self.exprs = [E.TryCast(ch[0], rt)]                                # agg.rs:190-197
            self.nullable = True
        elif f in (E.AGG_MAX, E.AGG_MIN):
            self.data_type = ch[0].data_type(input_schema)                     # agg.rs:198-205
            self.exprs = [ch[0]]
            self.nullable = True
        else:
            raise OracleError(f"aggregate function {f} is out of scope (SURVEY.md §2.1)")

    # ---- accumulators
    def create_acc(self):
        if self.function == E.AGG_COUNT:
            return _CountAcc()
        if self.function == E.AGG_AVG:
            return (_PrimAcc(self.data_type), _CountAcc())
        return _PrimAcc(self.data_type)

    @staticmethod
    def acc_resize(acc, n):
        if isinstance(acc, tuple):
            for a in acc: a.resize(n)
        else:
            acc.resize(n)

    @staticmethod
    def acc_len(acc):
        a = acc[0] if isinstance(acc, tuple) else acc
        return len(a.values)

    def _sum_update(self, acc: _PrimAcc, gids, arg: Col, rows):
        dt = self.data_type
        for g, r in zip(gids, rows):
            if arg.valid[r]:
                v = _np_scalar(dt, arg.values[r])
                acc.update_value(g, v, lambda cur, v=v: _add(dt, cur, v))      # sum.rs:103-109

    def _count_update(self, acc: _CountAcc, gids, args: List[Col], rows):
        for g, r in zip(gids, rows):
            add = 1 if all(a.valid[r] for a in args) else 0                   # count.rs:100-124
            acc.values[g] = wrap_i64(acc.values[g] + add)

    def _maxmin_update(self, acc: _PrimAcc, gids, arg: Col, rows):
        dt, ordv = self.data_type, ("Greater" if self.function == E.AGG_MAX else "Less")
        for g, r in zip(gids, rows):
            if arg.valid[r]:
                v = _np_scalar(dt, arg.values[r]) if dt.id != T.BOOL else bool(arg.values[r])
                acc.update_value(g, v, lambda cur, v=v: cur if _partial_cmp(dt, cur, v) == ordv else v)  # maxmin.rs:111-117

    def partial_update(self, acc, gids, args: List[Col], rows):
        f = self.function
        if f == E.AGG_COUNT:
            self._count_update(acc, gids, args, rows)
        elif f == E.AGG_SUM:
            self._sum_update(acc, gids, cast(args[0], self.data_type), rows)   # prepare_partial_args sum.rs:78-84
        elif f == E.AGG_AVG:
            a = cast(args[0], self.data_type)
            self._sum_update(acc[0], gids, a, rows)                            # avg.rs:109-123
            self._count_update(acc[1], gids, [a], rows)
        else:
            self._maxmin_update(acc, gids, args[0], rows)

    def partial_merge(self, acc, gids, macc, mrows):
        f, dt = self.function, self.data_type

        def merge_prim(a: _PrimAcc, m: _PrimAcc, fn):
            for g, r in zip(gids, mrows):
                if m.valids[r]:
                    v = m.values[r]
                    a.update_value(g, v, lambda cur, v=v: fn(cur, v))

        def merge_count(a: _CountAcc, m: _CountAcc):
            for g, r in zip(gids, mrows):
                a.values[g] = wrap_i64(a.values[g] + m.values[r])              # count.rs:128-149

        if f == E.AGG_COUNT:
            merge_count(acc, macc)
        elif f == E.AGG_SUM:
            merge_prim(acc, macc, lambda c, v: _add(dt, c, v))                 # sum.rs:117-145
        elif f == E.AGG_AVG:
            merge_prim(acc[0], macc[0], lambda c, v: _add(dt, c, v))
            merge_count(acc[1], macc[1])
        else:
            ordv = "Greater" if f == E.AGG_MAX else "Less"
            merge_prim(acc, macc, lambda c, v: c if _partial_cmp(dt, c, v) == ordv else v)

    # ---- freeze / unfreeze
    def freeze(self, acc, i) -> bytes:
        if isinstance(acc, tuple):
            return acc[0].freeze(i) + acc[1].freeze(i)                         # avg.rs:208-212
        return acc.freeze(i)

    def unfreeze_push(self, acc, buf, pos) -> int:
        if isinstance(acc, tuple):
            pos = acc[0].unfreeze_push(buf, pos)
            return acc[1].unfreeze_push(buf, pos)
        return acc.unfreeze_push(buf, pos)

    # ---- final
    def final_merge(self, acc, idx) -> Col:
        f = self.function
        if f == E.AGG_COUNT:
            return Col(T.int64, np.array([acc.values[i] for i in idx], np.int64), np.ones(len(idx), bool))
        if f == E.AGG_AVG:
            sums = acc[0].to_col(idx)
            counts = np.array([acc[1].values[i] for i in idx], np.int64)
            ok = sums.valid & (counts != 0)                                    # avg.rs:153-156
            if self.data_type.is_decimal:
                vals = np.empty(len(idx), object)
                for j in range(len(idx)):
                    if ok[j]:
                        s, c = int(sums.values[j]), int(counts[j])
                        q = s // c if c > 0 else -(s // -c)                     # checked_div_euclid (c>0 on this path)
                        vals[j] = q
                    else:
                        vals[j] = 0
                return Col(self.data_type, vals, ok)
            sv = np.array([float(v) for v in sums.values], np.float64) if len(idx) else np.zeros(0)
            vals = np.where(ok, sv / np.where(ok, counts, 1).astype(np.float64), 0.0)   # avg.rs:167-171
            return Col(T.float64, vals, ok)
        return acc.to_col(idx)

    def final_type(self) -> DataType:
        if self.function == E.AGG_AVG and not self.data_type.is_decimal:
            return T.float64
        return self.data_type


class AggExec:
    """datafusion-ext-plans/src/agg_exec.rs:59-323 + agg/agg_ctx.rs + agg/agg_table.rs (no-spill path;
    spilling changes only the emission order — SURVEY.md §8 A12)."""

    # native fallbacks when no JVM conf is reachable (agg/agg_ctx.rs:174-185)
    PARTIAL_SKIPPING_RATIO = 0.999
    PARTIAL_SKIPPING_MIN_ROWS = 20000

    def __init__(self, exec_mode: int, groupings: Sequence[E.GroupingExpr], aggs: Sequence[E.AggExpr],
                 supports_partial_skipping: bool, input_schema: Schema, batch_size: int = 10000):
        self.input_schema = input_schema
        self.groupings = list(groupings)
        self.agg_exprs = list(aggs)
        self.aggs = [Agg(a.agg, input_schema) for a in aggs]
        self.modes = [a.mode for a in aggs]
        self.supports_partial_skipping = supports_partial_skipping
        self.batch_size = batch_size
        self.need_partial_update = any(m == E.PARTIAL for m in self.modes)
        self.need_partial_merge = any(m != E.PARTIAL for m in self.modes)
        self.need_final_merge = any(m == E.FINAL for m in self.modes)
        assert not (self.need_final_merge and any(m != E.FINAL for m in self.modes))   # agg_ctx.rs:115
        gfields = [Field(g.field_name, g.expr.data_type(input_schema), g.expr.nullable(input_schema)) for g in groupings]
        if self.need_final_merge:
            afields = [Field(a.field_name, ag.final_type(), ag.nullable) for a, ag in zip(aggs, self.aggs)]
        else:
            afields = [Field(E.AGG_BUF_COLUMN_NAME, T.binary, False)]                   # agg_ctx.rs:139-141
        self.schema = Schema(gfields + afields)
        self.num_group_cols = len(gfields)

    # ---- helpers
    def _agg_args(self, batch: Batch) -> List[List[Col]]:
        out = []
        for ag, m in zip(self.aggs, self.modes):
            if m == E.PARTIAL:
                out.append([evaluate(e, batch).broadcast(batch.num_rows) for e in ag.exprs])
            else:
                out.append([])
        return out

    def _update(self, batch: Batch, accs, gids, nrec: int):
        """AggContext::update_batch_slice_to_acc_table (agg_ctx.rs:242-301)"""
        rows = range(batch.num_rows)
        for ag, acc in zip(self.aggs, accs):
            if Agg.acc_len(acc) < nrec:
                Agg.acc_resize(acc, nrec)                                      # ensure_size
        if self.need_partial_update:
            args = self._agg_args(batch)
            for ag, m, acc, a in zip(self.aggs, self.modes, accs, args):
                if m == E.PARTIAL:
                    ag.partial_update(acc, gids, a, rows)
        if self.need_partial_merge:
            bufcol = batch.cols[-1]                                            # always the LAST column (:280)
            maccs = [ag.create_acc() for ag in self.aggs]
            cursors = [0] * batch.num_rows
            for ag, m, macc in zip(self.aggs, self.modes, maccs):
                if m != E.PARTIAL:
                    for r in range(batch.num_rows):
                        cursors[r] = ag.unfreeze_push(macc, bufcol.values[r], cursors[r])
            for ag, m, acc, macc in zip(self.aggs, self.modes, accs, maccs):
                if m != E.PARTIAL:
                    ag.partial_merge(acc, gids, macc, rows)

    def _build_agg_cols(self, accs, idx) -> List[Col]:
        """AggContext::build_agg_columns (agg_ctx.rs:303-326)"""
        if self.need_final_merge:
            return [ag.final_merge(acc, idx) for ag, acc in zip(self.aggs, accs)]
        vals = np.empty(len(idx), object)
        for j, i in enumerate(idx):
            vals[j] = b"".join(ag.freeze(acc, i) for ag, acc in zip(self.aggs, accs))   # freeze_acc_table :407-426
        return [Col(T.binary, vals, np.ones(len(idx), bool))]

    def _key_cols(self, keys: List[tuple]) -> List[Col]:
        cols = []
        for k, f in enumerate(self.schema.fields[: self.num_group_cols]):
            vals, valid = _zeros(f.dtype, len(keys)), np.zeros(len(keys), bool)
            for j, key in enumerate(keys):
                if key[k] is not None:
                    vals[j] = key[k]; valid[j] = True
            cols.append(Col(f.dtype, vals, valid))
        return cols

    @staticmethod
    def _key_of(cols: List[Col], r: int) -> tuple:
        # group identity = arrow-row encoding of the key tuple (agg_ctx.rs:219-231): NULL is its own
        # group; floats are grouped by bit pattern after the row encoder's canonical form
        out = []
        for c in cols:
            if not c.valid[r]:
                out.append(None)
            else:
                v = c.values[r]
                out.append(v.item() if hasattr(v, "item") else v)
        return tuple(out)

    # ---- execution
    def execute(self, batches: Sequence[Batch]) -> List[Batch]:
        if not self.groupings:
            return self._execute_no_grouping(batches)
        out: List[Batch] = []
        table: Dict[tuple, int] = {}
        keys: List[tuple] = []
        accs = [ag.create_acc() for ag in self.aggs]
        num_input = 0
        skipping = False
        first_table = True
        for b in batches:
            if b.num_rows == 0:
                continue
            if skipping:
                out.append(self._process_partial_skipped(b))                   # agg_ctx.rs:428-462
                continue
            gcols = [evaluate(g.expr, b).broadcast(b.num_rows) for g in self.groupings]
            gids = []
            for r in range(b.num_rows):
                k = self._key_of(gcols, r)
                g = table.get(k)
                if g is None:
                    g = len(keys); table[k] = g; keys.append(k)
                gids.append(g)
            num_input += b.num_rows
            self._update(b, accs, gids, len(keys))
            # partial skipping by cardinality ratio (agg_table.rs:108-120, 447-463)
            if (self.supports_partial_skipping and first_table and len(keys) >= self.PARTIAL_SKIPPING_MIN_ROWS
                    and len(keys) / num_input > self.PARTIAL_SKIPPING_RATIO):
                out += self._output(keys, accs)
                table, keys, accs = {}, [], [ag.create_acc() for ag in self.aggs]
                skipping = True
        out += self._output(keys, accs)
        return out

    def _output(self, keys, accs) -> List[Batch]:
        """AggTable::output, no-spill branch: chunks emitted last-to-first (agg_table.rs:163-207)"""
        n = len(keys)
        out = []
        step = self.batch_size
        for begin in reversed(range(0, n, step)):
            idx = list(range(begin, min(begin + step, n)))
            cols = self._key_cols([keys[i] for i in idx]) + self._build_agg_cols(accs, idx)
            out.append(Batch(self.schema, cols, len(idx)))
        return out

    def _process_partial_skipped(self, b: Batch) -> Batch:
        accs = [ag.create_acc() for ag in self.aggs]
        for acc in accs:
            Agg.acc_resize(acc, b.num_rows)
        self._update(b, accs, list(range(b.num_rows)), b.num_rows)
        gcols = [evaluate(g.expr, b).broadcast(b.num_rows) for g in self.groupings]
        gcols = [Col(c.dtype, c.values, c.valid) for c in gcols]
        return Batch(self.schema, gcols + self._build_agg_cols(accs, list(range(b.num_rows))), b.num_rows)

    def _execute_no_grouping(self, batches) -> List[Batch]:
        """execute_agg_no_grouping (agg_exec.rs:280-323): always exactly one output row"""
        accs = [ag.create_acc() for ag in self.aggs]
        for acc in accs:
            Agg.acc_resize(acc, 1)
        for b in batches:
            if b.num_rows:
                self._update(b, accs, [0] * b.num_rows, 1)
        return [Batch(self.schema, self._build_agg_cols(accs, [0]), 1)]


# =================================================================================================
# Spark-compatible murmur3 + pmod partition ids (the multi-GPU exchange key)
# =================================================================================================

def _u32(x): return x & 0xFFFFFFFF


def _rotl(x, r): return _u32((x << r) | (x >> (32 - r)))


def _mix_k1(k1):
    k1 = _u32(k1 * 0xcc9e2d51); k1 = _rotl(k1, 15); return _u32(k1 * 0x1b873593)


def _mix_h1(h1, k1):
    h1 ^= k1; h1 = _rotl(h1, 13); return _u32(h1 * 5 + 0xe6546b64)


def _fmix(h1, length):
    h1 ^= length; h1 ^= h1 >> 16; h1 = _u32(h1 * 0x85ebca6b); h1 ^= h1 >> 13; h1 = _u32(h1 * 0xc2b2ae35); h1 ^= h1 >> 16
    return h1


def _to_i32(x): return x - (1 << 32) if x >> 31 else x


def murmur3_bytes(data: bytes, seed: int) -> int:
    """spark_compatible_murmur3_hash (datafusion-ext-commons/src/hash/mur.rs:19-30)"""
    h1 = _u32(seed)
    n = len(data)
    aligned = n - n % 4
    for i in range(0, aligned, 4):
        h1 = _mix_h1(h1, _mix_k1(int.from_bytes(data[i:i + 4], "little")))
    for b in data[aligned:]:
        sb = b - 256 if b >= 128 else b                                # `b as i8 as i32`
        h1 = _mix_h1(h1, _mix_k1(_u32(sb)))
    return _to_i32(_fmix(h1, n))


def murmur3_long(v: int, seed: int) -> int:
    """hash_long (mur.rs:75-87) == murmur3_bytes(le_bytes(v))"""
    return murmur3_bytes((v & ((1 << 64) - 1)).to_bytes(8, "little"), seed)


def create_murmur3_hashes(cols: Sequence[Col], n: int, seed: int = 42) -> np.ndarray:
    """create_murmur3_hashes / hash_array (spark_hash.rs:28-32, 62-200): chained over columns,
    NULL leaves the running hash unchanged; int8/16/32/date32 hash as 4 LE bytes, int64/ts as 8,
    f32/f64 by their bit patterns, bool as u32 0/1, decimal128 as 16 LE bytes."""
    h = [seed] * n
    for c in cols:
        w = {T.INT8: 4, T.INT16: 4, T.INT32: 4, T.DATE32: 4, T.INT64: 8, T.TIMESTAMP_US: 8,
             T.FLOAT32: 4, T.FLOAT64: 8, T.BOOL: 4, T.DECIMAL128: 16, T.BINARY: 0}[c.dtype.id]
        for i in range(n):
            if not c.valid[i]:
                continue
            v = c.values[i]
            if c.dtype.id == T.BINARY:
                data = bytes(v)
            elif c.dtype.id == T.FLOAT32:
                data = struct.pack("<f", v)
            elif c.dtype.id == T.FLOAT64:
                data = struct.pack("<d", v)
            else:
                data = (int(v) & ((1 << (8 * w)) - 1)).to_bytes(w, "little")
            h[i] = murmur3_bytes(data, h[i])
    return np.array(h, np.int32)


def partition_ids(hashes: np.ndarray, num_partitions: int) -> np.ndarray:
    """evaluate_partition_ids (datafusion-ext-plans/src/shuffle/mod.rs:178-188): pmod = rem_euclid"""
    return np.mod(hashes.astype(np.int64), num_partitions).astype(np.uint32)


# =================================================================================================
# helpers for tests: order-insensitive multiset comparison (assert_batches_sorted_eq!)
# =================================================================================================

def rows_multiset(batches: Sequence[Batch]) -> Dict[tuple, int]:
    out: Dict[tuple, int] = {}
    for b in batches:
        for r in range(b.num_rows):
            key = []
            for c in b.cols:
                if not c.valid[r]:
                    key.append(None)
                else:
                    v = c.values[r]
                    v = v.item() if hasattr(v, "item") else v
                    if isinstance(v, float):
                        v = struct.pack("<d", v)                      # bit-exact float identity
                    key.append(v)
            key = tuple(key)
            out[key] = out.get(key, 0) + 1
    return out


def concat_batches(schema: Schema, batches: Sequence[Batch]) -> Batch:
    if not batches:
        return Batch.empty(schema)
    cols = []
    for i in range(len(schema)):
        cols.append(Col(schema[i].dtype, np.concatenate([b.cols[i].values for b in batches]),
                        np.concatenate([b.cols[i].valid for b in batches])))
    return Batch(schema, cols, sum(b.num_rows for b in batches))
