"""Arrow data types of the hot path (Filter/Project/Agg over fixed-width columns).

Mirrors the `ArrowType` subset of the reference plan-serde
(native-engine/auron-serde/proto/auron.proto:860-896) that the Spark converter emits
for fixed-width columns (spark-extension/.../NativeConverters.scala:117-144).
Pure data: no compute lives here.
"""
from __future__ import annotations

from dataclasses import dataclass

# type ids shared with the C ABI (include/blaze_b200.h: b200q_type_id)
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIMESTAMP_US, DECIMAL128, BINARY, NULLTYPE, UTF8 = range(13)

_NAMES = {
    BOOL: "bool", INT8: "int8", INT16: "int16", INT32: "int32", INT64: "int64",
    FLOAT32: "float32", FLOAT64: "float64", DATE32: "date32", TIMESTAMP_US: "timestamp[us]",
    DECIMAL128: "decimal128", BINARY: "binary", NULLTYPE: "null", UTF8: "utf8",
}


@dataclass(frozen=True)
class DataType:
    id: int
    precision: int = 0   # decimal128 only
    scale: int = 0       # decimal128 only

    def __str__(self) -> str:
        if self.id == DECIMAL128:
            return f"decimal128({self.precision},{self.scale})"
        return _NAMES[self.id]

    @property
    def is_integer(self) -> bool:
        return self.id in (INT8, INT16, INT32, INT64)

    @property
    def is_float(self) -> bool:
        return self.id in (FLOAT32, FLOAT64)

    @property
    def is_decimal(self) -> bool:
        return self.id == DECIMAL128

    @property
    def is_numeric(self) -> bool:
        return self.is_integer or self.is_float or self.is_decimal

    @property
    def bit_width(self) -> int:
        return {BOOL: 1, INT8: 8, INT16: 16, INT32: 32, INT64: 64, FLOAT32: 32, FLOAT64: 64,
                DATE32: 32, TIMESTAMP_US: 64, DECIMAL128: 128}.get(self.id, 0)


bool_ = DataType(BOOL)
int8 = DataType(INT8)
int16 = DataType(INT16)
int32 = DataType(INT32)
int64 = DataType(INT64)
float32 = DataType(FLOAT32)
float64 = DataType(FLOAT64)
date32 = DataType(DATE32)
timestamp_us = DataType(TIMESTAMP_US)
binary = DataType(BINARY)
utf8 = DataType(UTF8)
null = DataType(NULLTYPE)


def decimal128(precision: int, scale: int) -> DataType:
    assert 1 <= precision <= 38
    return DataType(DECIMAL128, precision, scale)


@dataclass(frozen=True)
class Field:
    name: str
    dtype: DataType
    nullable: bool = True


@dataclass(frozen=True)
class Schema:
    fields: tuple

    def __init__(self, fields):
        object.__setattr__(self, "fields", tuple(fields))

    def index_of(self, name: str) -> int:
        for i, f in enumerate(self.fields):
            if f.name == name:
                return i
        raise KeyError(f"column {name!r} not in schema {[f.name for f in self.fields]}")

    def __len__(self):
        return len(self.fields)

    def __iter__(self):
        return iter(self.fields)

    def __getitem__(self, i):
        return self.fields[i]


# ---- pyarrow bridges (pyarrow is only a container/FFI carrier here) -----------------------------

def from_arrow_type(t) -> DataType:
    import pyarrow as pa
    if pa.types.is_boolean(t): return bool_
    if pa.types.is_int8(t): return int8
    if pa.types.is_int16(t): return int16
    if pa.types.is_int32(t): return int32
    if pa.types.is_int64(t): return int64
    if pa.types.is_float32(t): return float32
    if pa.types.is_float64(t): return float64
    if pa.types.is_date32(t): return date32
    if pa.types.is_timestamp(t):
        if t.unit != "us":
            raise TypeError(f"only timestamp[us] is on the hot path, got {t}")
        return timestamp_us
    if pa.types.is_decimal128(t): return decimal128(t.precision, t.scale)
    if pa.types.is_binary(t): return binary
    if pa.types.is_string(t): return utf8
    if pa.types.is_null(t): return null
    raise TypeError(f"unsupported arrow type on the hot path: {t}")


def to_arrow_type(dt: DataType):
    import pyarrow as pa
    return {
        BOOL: pa.bool_(), INT8: pa.int8(), INT16: pa.int16(), INT32: pa.int32(), INT64: pa.int64(),
        FLOAT32: pa.float32(), FLOAT64: pa.float64(), DATE32: pa.date32(),
        TIMESTAMP_US: pa.timestamp("us"), BINARY: pa.binary(), NULLTYPE: pa.null(), UTF8: pa.string(),
    }[dt.id] if dt.id != DECIMAL128 else pa.decimal128(dt.precision, dt.scale)


def from_arrow_schema(s) -> Schema:
    return Schema(Field(f.name, from_arrow_type(f.type), f.nullable) for f in s)


def to_arrow_schema(s: Schema):
    import pyarrow as pa
    return pa.schema([pa.field(f.name, to_arrow_type(f.dtype), f.nullable) for f in s])
