"""CPU oracle for the Utf8 slice of the hot path: what the reference computes for string columns in FilterExec / ProjectExec
and for the string expressions, restated from the published semantics (not from the reference's source):

- comparisons Eq/NotEq/Lt/LtEq/Gt/GtEq over Utf8: arrow-rs `cmp` kernels order Utf8 by unsigned byte-lexicographic order of the
  UTF-8 bytes, a proper prefix first (Python `bytes` ordering is exactly that); NULL on either side gives NULL;
- StringStartsWithExpr / StringEndsWithExpr / StringContainsExpr (datafusion-ext-exprs/src/string_starts_with.rs:80-97,
  string_ends_with.rs, string_contains.rs): Rust `str::starts_with` / `ends_with` / `contains` per row, NULL in -> NULL out, an
  empty pattern matches every non-NULL string;
- InList (DataFusion `InListExpr`): NULL operand -> NULL; found -> true (false when negated); not found and a NULL item in the
  list -> NULL; otherwise false (true when negated);
- TryCast(Utf8 -> Int8/16/32/64): the reference's port of Spark `UTF8String.toLong` (datafusion-ext-commons/src/arrow/cast.rs:287-361).

Values are Python objects: Utf8 as `bytes`, integers as `int`, booleans as `bool`, NULL as None.  Rows of non-string columns are
taken as they are; the numeric expression semantics live in oracle/blaze_oracle.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

from blaze_b200 import exprs as E, types as T


def to_long(s: Optional[bytes], bits: int = 64) -> Optional[int]:
    """Spark UTF8String.toLong/toInt as ported at cast.rs:287-361: no trimming; an optional leading '+'/'-' (a lone sign is NULL);
    digits up to an optional '.', after which only digits may follow (they are dropped); any other byte, an empty string or a value
    outside the target width is NULL.  So "." -> 0, "-." -> 0, "1." -> 1, " 1" -> NULL."""
    if s is None or len(s) == 0:
        return None
    neg = s[0:1] == b"-"
    i = 0
    if neg or s[0:1] == b"+":
        i = 1
        if len(s) == 1:
            return None
    digits = []
    while i < len(s):
        b = s[i]
        i += 1
        if b == ord("."):
            break
        if not (ord("0") <= b <= ord("9")):
            return None
        digits.append(b - ord("0"))
    if any(not (ord("0") <= b <= ord("9")) for b in s[i:]):
        return None
    v = 0
    for d in digits:
        v = v * 10 + d
    v = -v if neg else v
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    return v if lo <= v <= hi else None


def _cmp(op: str, a, b) -> bool:
    return {"Eq": a == b, "NotEq": a != b, "Lt": a < b, "LtEq": a <= b, "Gt": a > b, "GtEq": a >= b}[op]


def _and(a, b):
    if a is False or b is False:
        return False
    if a is None or b is None:
        return None
    return True


def _or(a, b):
    if a is True or b is True:
        return True
    if a is None or b is None:
        return None
    return False


def _lit(value, dt: T.DataType):
    if value is None:
        return None
    if dt.id == T.UTF8:
        return value.encode() if isinstance(value, str) else bytes(value)
    return value


def evaluate(expr: E.Expr, cols: Dict[str, list], schema: T.Schema, n: int) -> list:
    """expr over `n` rows of `cols` (column name -> list of Python values) -> list of Python values"""
    if isinstance(expr, E.Column):
        return list(cols[expr.name])
    if isinstance(expr, E.Literal):
        return [_lit(expr.value, expr.dtype)] * n
    if isinstance(expr, E.BinaryExpr):
        l, r = evaluate(expr.left, cols, schema, n), evaluate(expr.right, cols, schema, n)
        if expr.op == "And":
            return [_and(a, b) for a, b in zip(l, r)]
        if expr.op == "Or":
            return [_or(a, b) for a, b in zip(l, r)]
        if expr.op in E.COMPARISONS:
            return [None if a is None or b is None else _cmp(expr.op, a, b) for a, b in zip(l, r)]
        raise NotImplementedError(f"string oracle: operator {expr.op}")
    if isinstance(expr, E.SCAnd):
        return [_and(a, b) for a, b in zip(evaluate(expr.left, cols, schema, n), evaluate(expr.right, cols, schema, n))]
    if isinstance(expr, E.SCOr):
        return [_or(a, b) for a, b in zip(evaluate(expr.left, cols, schema, n), evaluate(expr.right, cols, schema, n))]
    if isinstance(expr, E.IsNull):
        return [v is None for v in evaluate(expr.expr, cols, schema, n)]
    if isinstance(expr, E.IsNotNull):
        return [v is not None for v in evaluate(expr.expr, cols, schema, n)]
    if isinstance(expr, E.Not):
        return [None if v is None else not v for v in evaluate(expr.expr, cols, schema, n)]
    if isinstance(expr, E.StringMatch):
        p = expr.pattern.encode()
        f = {"StartsWith": lambda s: s.startswith(p), "EndsWith": lambda s: s.endswith(p), "Contains": lambda s: p in s}[expr.kind]
        return [None if v is None else f(v) for v in evaluate(expr.expr, cols, schema, n)]
    if isinstance(expr, E.InList):
        x = evaluate(expr.expr, cols, schema, n)
        items = [_lit(it.value, it.dtype) for it in expr.list]
        has_null = any(it is None for it in items)
        vals = set(it for it in items if it is not None)
        out = []
        for v in x:
            if v is None:
                out.append(None)
            elif v in vals:
                out.append(not expr.negated)
            else:
                out.append(None if has_null else expr.negated)
        return out
    if isinstance(expr, E.TryCast):
        src, to = expr.expr.data_type(schema), expr.dtype
        v = evaluate(expr.expr, cols, schema, n)
        if src == to:
            return v
        if src.id == T.UTF8 and to.is_integer:
            return [to_long(s, to.bit_width) for s in v]
        raise NotImplementedError(f"string oracle: TryCast {src} -> {to}")
    raise NotImplementedError(f"string oracle: {type(expr).__name__}")


def columns_of(batches: Sequence) -> Dict[str, list]:
    """pyarrow RecordBatches -> column name -> Python values (Utf8 as bytes)"""
    import pyarrow as pa
    out: Dict[str, list] = {}
    if not batches:
        return out
    for name in batches[0].schema.names:
        vals: List = []
        for b in batches:
            c = b.column(name)
            if pa.types.is_string(c.type):
                vals += [None if v is None else v.encode() for v in c.to_pylist()]
            else:
                vals += c.to_pylist()
        out[name] = vals
    return out


def filter_project(predicates: Sequence[E.Expr], projections: Optional[Sequence], schema: T.Schema, batches: Sequence) -> List[tuple]:
    """FilterExec (rows where every predicate is true; NULL filters the row out, filter_exec.rs) then ProjectExec -> ordered rows"""
    cols = columns_of(batches)
    n = sum(b.num_rows for b in batches)
    keep = [True] * n
    for p in predicates:
        keep = [k and v is True for k, v in zip(keep, evaluate(p, cols, schema, n))]
    exprs = [e for e, _ in projections] if projections is not None else [E.Column(f.name) for f in schema]
    outs = [evaluate(e, cols, schema, n) for e in exprs]
    return [tuple(o[i] for o in outs) for i in range(n) if keep[i]]


def rows_of(batches: Sequence) -> List[tuple]:
    """pyarrow RecordBatches -> ordered rows of Python values (Utf8 as bytes)"""
    cols = columns_of(batches)
    names = batches[0].schema.names if batches else []
    n = sum(b.num_rows for b in batches)
    return [tuple(cols[c][i] for c in names) for i in range(n)]
