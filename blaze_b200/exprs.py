"""Physical expressions of the hot path — the host-side mirror of what
`try_parse_physical_expr` builds (native-engine/auron-serde/src/from_proto.rs:839-1026).

These are plain descriptions (no evaluation code): they are serialised to the reference's
protobuf (`blaze_b200.proto`) and shipped through the C ABI; the CPU oracle under `oracle/`
walks the same trees. Type / nullability rules follow DataFusion 49 `PhysicalExpr::data_type`
/ `nullable` (third-party, un-vendored: SURVEY.md §8c) and the reference's own `TryCastExpr`
(native-engine/datafusion-ext-exprs/src/cast.rs:56-67, always nullable).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Optional, Sequence, Tuple

from . import types as T
from .types import DataType, Schema

COMPARISONS = ("Eq", "NotEq", "Lt", "LtEq", "Gt", "GtEq")
ARITHMETIC = ("Plus", "Minus", "Multiply", "Divide", "Modulo")
LOGICAL = ("And", "Or")
BITWISE = ("BitwiseAnd", "BitwiseOr", "BitwiseXor")
# the full operator-name table accepted by the reference: auron-serde/src/lib.rs:70-102
BINARY_OPS = COMPARISONS + ARITHMETIC + LOGICAL + BITWISE


class Expr:
    def data_type(self, schema: Schema) -> DataType:
        raise NotImplementedError

    def nullable(self, schema: Schema) -> bool:
        raise NotImplementedError

    def children(self) -> Sequence["Expr"]:
        return ()


@dataclass(frozen=True)
class Column(Expr):
    """`PhysicalColumn{name}` — resolved BY NAME against the child schema (from_proto.rs:850)."""
    name: str

    def data_type(self, schema):
        return schema[schema.index_of(self.name)].dtype

    def nullable(self, schema):
        return schema[schema.index_of(self.name)].nullable


@dataclass(frozen=True)
class BoundReference(Expr):
    """`BoundReference{index,data_type,nullable}` — positional (from_proto.rs:852-855)."""
    index: int
    dtype: Optional[DataType] = None
    is_nullable: bool = True

    def data_type(self, schema):
        return schema[self.index].dtype

    def nullable(self, schema):
        return schema[self.index].nullable


@dataclass(frozen=True)
class Literal(Expr):
    """`ScalarValue{ipc_bytes}`: value None = typed NULL. Decimal values are unscaled ints."""
    value: Any
    dtype: DataType

    def data_type(self, schema):
        return self.dtype

    def nullable(self, schema):
        return self.value is None


@dataclass(frozen=True)
class BinaryExpr(Expr):
    left: Expr
    op: str
    right: Expr

    def __post_init__(self):
        if self.op not in BINARY_OPS:
            raise ValueError(f"Unsupported binary operator {self.op!r}")

    def children(self):
        return (self.left, self.right)

    def data_type(self, schema):
        lt, rt = self.left.data_type(schema), self.right.data_type(schema)
        if self.op in COMPARISONS or self.op in LOGICAL:
            return T.bool_
        if lt.is_decimal and rt.is_decimal:
            return decimal_result_type(self.op, lt, rt)
        if lt != rt:
            raise TypeError(f"binary {self.op}: operand types differ: {lt} vs {rt} "
                            "(the Spark converter inserts the casts; arrow kernels do not coerce)")
        return lt

    def nullable(self, schema):
        return self.left.nullable(schema) or self.right.nullable(schema)


def decimal_result_type(op: str, l: DataType, r: DataType) -> DataType:
    """arrow-arith 55.2 `decimal_op` result types for Decimal128 (un-vendored; documented rules)."""
    if op in ("Plus", "Minus"):
        s = max(l.scale, r.scale)
        p = min(38, max(l.precision - l.scale, r.precision - r.scale) + s + 1)
        return T.decimal128(p, s)
    raise TypeError(f"decimal {op} is not on the hot path (round 1)")


@dataclass(frozen=True)
class IsNull(Expr):
    expr: Expr
    def children(self): return (self.expr,)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return False


@dataclass(frozen=True)
class IsNotNull(Expr):
    expr: Expr
    def children(self): return (self.expr,)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return False


@dataclass(frozen=True)
class Not(Expr):
    expr: Expr
    def children(self): return (self.expr,)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return self.expr.nullable(schema)


@dataclass(frozen=True)
class Negative(Expr):
    expr: Expr
    def children(self): return (self.expr,)
    def data_type(self, schema): return self.expr.data_type(schema)
    def nullable(self, schema): return self.expr.nullable(schema)


@dataclass(frozen=True)
class Cast(Expr):
    """DataFusion `CastExpr` (PhysicalCastNode): nullable follows the child."""
    expr: Expr
    dtype: DataType
    def children(self): return (self.expr,)
    def data_type(self, schema): return self.dtype
    def nullable(self, schema): return self.expr.nullable(schema)


@dataclass(frozen=True)
class TryCast(Expr):
    """Reference `TryCastExpr` (datafusion-ext-exprs/src/cast.rs:33-101): always nullable."""
    expr: Expr
    dtype: DataType
    def children(self): return (self.expr,)
    def data_type(self, schema): return self.dtype
    def nullable(self, schema): return True


@dataclass(frozen=True)
class Case(Expr):
    """`CASE [expr] WHEN w THEN t ... [ELSE e] END` (PhysicalCaseNode)."""
    expr: Optional[Expr]
    when_then: Tuple[Tuple[Expr, Expr], ...]
    else_expr: Optional[Expr] = None

    def __init__(self, expr, when_then, else_expr=None):
        object.__setattr__(self, "expr", expr)
        object.__setattr__(self, "when_then", tuple((w, t) for w, t in when_then))
        object.__setattr__(self, "else_expr", else_expr)

    def children(self):
        out = [] if self.expr is None else [self.expr]
        for w, t in self.when_then:
            out += [w, t]
        if self.else_expr is not None:
            out.append(self.else_expr)
        return tuple(out)

    def data_type(self, schema):
        # DataFusion CaseExpr::data_type: first non-Null THEN type, else the ELSE type
        for _, t in self.when_then:
            dt = t.data_type(schema)
            if dt.id != T.NULLTYPE:
                return dt
        if self.else_expr is not None:
            return self.else_expr.data_type(schema)
        return T.null

    def nullable(self, schema):
        # DataFusion CaseExpr::nullable: any THEN nullable, or no ELSE, or ELSE nullable
        if any(t.nullable(schema) for _, t in self.when_then):
            return True
        return True if self.else_expr is None else self.else_expr.nullable(schema)


@dataclass(frozen=True)
class InList(Expr):
    expr: Expr
    list: Tuple[Expr, ...]
    negated: bool = False

    def __init__(self, expr, list, negated=False):
        object.__setattr__(self, "expr", expr)
        object.__setattr__(self, "list", tuple(list))
        object.__setattr__(self, "negated", bool(negated))

    def children(self): return (self.expr,) + self.list
    def data_type(self, schema): return T.bool_
    def nullable(self, schema):
        return self.expr.nullable(schema) or any(e.nullable(schema) for e in self.list)


@dataclass(frozen=True)
class SCAnd(Expr):
    """fork-only short-circuit AND (from_proto.rs:1010-1014): same truth table as Kleene And."""
    left: Expr
    right: Expr
    def children(self): return (self.left, self.right)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return self.left.nullable(schema) or self.right.nullable(schema)


@dataclass(frozen=True)
class SCOr(Expr):
    left: Expr
    right: Expr
    def children(self): return (self.left, self.right)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return self.left.nullable(schema) or self.right.nullable(schema)


@dataclass(frozen=True)
class StringMatch(Expr):
    """`StringStartsWithExprNode{expr, prefix}` / `StringEndsWithExprNode{expr, suffix}` / `StringContainsExprNode{expr, infix}`
    (auron.proto:339-352): Boolean, always nullable (datafusion-ext-exprs/src/string_starts_with.rs:73-79)."""
    kind: str            # "StartsWith" | "EndsWith" | "Contains"
    expr: Expr
    pattern: str

    def __post_init__(self):
        if self.kind not in STRING_MATCH_KINDS:
            raise ValueError(f"unknown string match {self.kind!r}")

    def children(self): return (self.expr,)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return True


STRING_MATCH_KINDS = ("StartsWith", "EndsWith", "Contains")


def StartsWith(expr: Expr, prefix: str) -> StringMatch: return StringMatch("StartsWith", expr, prefix)
def EndsWith(expr: Expr, suffix: str) -> StringMatch: return StringMatch("EndsWith", expr, suffix)
def Contains(expr: Expr, infix: str) -> StringMatch: return StringMatch("Contains", expr, infix)


# Spark ext functions on the hot path (datafusion-ext-functions/src/lib.rs:34-68)
SPARK_EXT_FUNCTIONS = ("UnscaledValue", "MakeDecimal", "CheckOverflow", "NullIfZero", "NullIf",
                       "NormalizeNanAndZero", "Placeholder", "XxHash64")


@dataclass(frozen=True)
class ScalarFunction(Expr):
    """`PhysicalScalarFunctionNode{fun=SparkExtFunctions,name,args,return_type}`; result field is
    declared nullable=true by the reference (from_proto.rs:965-972)."""
    name: str
    args: Tuple[Expr, ...]
    return_type: DataType

    def __init__(self, name, args, return_type):
        object.__setattr__(self, "name", name)
        object.__setattr__(self, "args", tuple(args))
        object.__setattr__(self, "return_type", return_type)

    def children(self): return self.args
    def data_type(self, schema): return self.return_type
    def nullable(self, schema): return True


def XxHash64(*args: Expr) -> ScalarFunction:
    """Spark's XxHash64(children, 42) (spark_hash.rs spark_xxhash64): h = 42, then h = xxhash64(child, h) per child; a NULL
    child leaves h unchanged, so the result is never NULL."""
    return ScalarFunction("XxHash64", args, T.int64)


@dataclass(frozen=True)
class ScalarSubquery(Expr):
    """`PhysicalSparkScalarSubqueryWrapperExprNode{serialized, return_type, return_nullable}` (auron.proto:318-322): a scalar
    subquery the JVM evaluates.  On the device path it is accepted only as the bloom filter of BloomFilterMightContain, and
    the host's resolver (native.set_scalar_subquery_resolver) turns `serialized` into the value at op create."""
    serialized: bytes
    return_type: DataType = T.binary
    return_nullable: bool = True

    def data_type(self, schema): return self.return_type
    def nullable(self, schema): return self.return_nullable


@dataclass(frozen=True)
class BloomFilterMightContain(Expr):
    """`BloomFilterMightContainExprNode{uuid, bloom_filter_expr, value_expr}` (bloom_filter_might_contain.rs): whether the
    Spark bloom filter (a Binary literal, or a ScalarSubquery) might contain the Int8..Int64 value.  A NULL filter gives false
    for every row; a NULL value gives NULL."""
    bloom_filter: Expr
    value: Expr
    uuid: str = ""

    def children(self): return (self.bloom_filter, self.value)
    def data_type(self, schema): return T.bool_
    def nullable(self, schema): return True


# ---- aggregate descriptions ----------------------------------------------------------------------

# AggFunction enum values (auron.proto:127-141)
AGG_MIN, AGG_MAX, AGG_SUM, AGG_AVG, AGG_COUNT = 0, 1, 2, 3, 4
AGG_FIRST, AGG_FIRST_IGNORES_NULL = 7, 8
AGG_BLOOM_FILTER = 9             # children: value, Literal(estimated_num_items), Literal(num_bits); the state and result are Binary
AGG_NAMES = {AGG_MIN: "Min", AGG_MAX: "Max", AGG_SUM: "Sum", AGG_AVG: "Avg", AGG_COUNT: "Count",
             AGG_FIRST: "First", AGG_FIRST_IGNORES_NULL: "FirstIgnoresNull", AGG_BLOOM_FILTER: "BloomFilter"}

# AggMode (auron.proto:692-696) / AggExecMode (:687-690)
PARTIAL, PARTIAL_MERGE, FINAL = 0, 1, 2
HASH_AGG, SORT_AGG = 0, 1

# name of the single Binary accumulator column of non-final agg output
# (datafusion-ext-plans/src/agg/mod.rs:37; NativeAggBase.scala:211-212)
AGG_BUF_COLUMN_NAME = "#9223372036854775807"


@dataclass(frozen=True)
class AggFunctionExpr:
    """`PhysicalAggExprNode{agg_function, children, return_type}` — what `create_agg` consumes
    (datafusion-ext-plans/src/agg/agg.rs:171-205)."""
    function: int
    children: Tuple[Expr, ...]
    return_type: DataType

    def __init__(self, function, children, return_type):
        object.__setattr__(self, "function", function)
        object.__setattr__(self, "children", tuple(children))
        object.__setattr__(self, "return_type", return_type)


# WindowFunction / WindowFunctionType (auron.proto:121-125, 556-559)
ROW_NUMBER, RANK, DENSE_RANK = 0, 1, 2
WINDOW_FUNC, WINDOW_AGG = 0, 1


@dataclass(frozen=True)
class WindowExpr:
    """`WindowExprNode{field, return_type, func_type, window_func, agg_func, children}` — WindowExpr::new(func, children,
    field, return_type) (datafusion-ext-plans/src/window/mod.rs).  Rank-like: func_type WINDOW_FUNC, window_func one of
    ROW_NUMBER / RANK / DENSE_RANK; aggregates: func_type WINDOW_AGG, agg_func an AGG_* code over `children`."""
    field: "T.Field"
    func_type: int
    window_func: int = ROW_NUMBER
    agg_func: int = 0
    children: Tuple[Expr, ...] = ()
    return_type: Optional[DataType] = None

    def __init__(self, field, func_type, window_func=ROW_NUMBER, agg_func=0, children=(), return_type=None):
        object.__setattr__(self, "field", field)
        object.__setattr__(self, "func_type", func_type)
        object.__setattr__(self, "window_func", window_func)
        object.__setattr__(self, "agg_func", agg_func)
        object.__setattr__(self, "children", tuple(children))
        object.__setattr__(self, "return_type", return_type if return_type is not None else field.dtype)

    @classmethod
    def rank_like(cls, name: str, window_func: int, nullable: bool = False):
        return cls(T.Field(name, T.int32, nullable), WINDOW_FUNC, window_func=window_func)

    @classmethod
    def agg(cls, name: str, agg_func: int, children, return_type: DataType, nullable: bool = True):
        return cls(T.Field(name, return_type, nullable), WINDOW_AGG, agg_func=agg_func, children=children, return_type=return_type)


@dataclass(frozen=True)
class GroupingExpr:
    field_name: str
    expr: Expr


@dataclass(frozen=True)
class AggExpr:
    field_name: str
    mode: int
    agg: AggFunctionExpr


def placeholder(dtype: DataType = T.null) -> Expr:
    """children of PartialMerge/Final aggs are placeholders that must never be evaluated
    (NativeAggBase.scala:241-282; datafusion-ext-functions/src/lib.rs:36)."""
    return ScalarFunction("Placeholder", (), dtype)
