"""FIRST / FIRST_IGNORES_NULL restated row by row (datafusion-ext-plans/src/agg/first.rs, first_ignores_null.rs), on top of the
AggExec of oracle/blaze_oracle.py: `Agg` instances of the other five functions are used as they are.

- FIRST: a group takes the value of the first row it sees, NULL or not, and sets its flag; later rows never replace it.
  Merge: the first state row whose flag is set wins, and its value may be NULL.  State (acc.rs): the value as an
  AccPrimColumn (`[u8 valid][LE value]`, or the AccBooleanColumn byte for Boolean values) followed by the flag as an
  AccBooleanColumn byte (0 unset, 1 + value if set, so a set flag is 2; any non-zero byte reads back as set).
- FIRST_IGNORES_NULL: the first non-NULL value; merge: the first state row with a valid value.  State: the value only.

"First" is arrival order: batches in the order given, rows in batch order.
"""
import os
import sys
from typing import List

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from blaze_b200 import exprs as E, types as T  # noqa: E402
from blaze_b200.types import Field, Schema  # noqa: E402
from oracle import blaze_oracle as O  # noqa: E402

FIRST_FNS = (E.AGG_FIRST, E.AGG_FIRST_IGNORES_NULL)


class _FlagAcc:
    """the AccBooleanColumn of FIRST's flags (acc.rs:101-241): None unset, True set"""

    def __init__(self):
        self.values: List[bool] = []

    def resize(self, n):
        while len(self.values) < n:
            self.values.append(False)
        del self.values[n:]

    def freeze(self, i) -> bytes:
        return b"\x02" if self.values[i] else b"\x00"

    def unfreeze_push(self, buf, pos):
        self.values.append(buf[pos] != 0)
        return pos + 1


class FirstAgg(O.Agg):
    def __init__(self, fexpr: E.AggFunctionExpr, input_schema: Schema):
        f, ch, rt = fexpr.function, list(fexpr.children), fexpr.return_type
        assert f in FIRST_FNS
        self.function = f
        dt = ch[0].data_type(input_schema)
        self.data_type = rt if dt == T.null else dt                    # merge side: a Placeholder of type Null
        if self.data_type.id in (T.UTF8, T.BINARY):
            raise O.OracleError("FIRST over Utf8 / Binary is out of scope")
        self.exprs = [ch[0]]
        self.nullable = True

    def create_acc(self):
        if self.function == E.AGG_FIRST:
            return (O._PrimAcc(self.data_type), _FlagAcc())
        return O._PrimAcc(self.data_type)

    def _value(self, col: O.Col, r):
        if self.data_type.id == T.BOOL:
            return bool(col.values[r])
        return O._np_scalar(self.data_type, col.values[r])

    def partial_update(self, acc, gids, args: List[O.Col], rows):
        arg = args[0]
        for g, r in zip(gids, rows):
            if self.function == E.AGG_FIRST:
                vals, flags = acc
                if not flags.values[g]:                                  # first.rs: any row, NULL or not
                    vals.valids[g] = bool(arg.valid[r])
                    vals.values[g] = self._value(arg, r) if arg.valid[r] else vals.values[g]
                    flags.values[g] = True
            elif not acc.valids[g] and arg.valid[r]:                     # first_ignores_null.rs: a valid value
                acc.values[g] = self._value(arg, r); acc.valids[g] = True

    def partial_merge(self, acc, gids, macc, mrows):
        for g, r in zip(gids, mrows):
            if self.function == E.AGG_FIRST:
                vals, flags = acc
                mvals, mflags = macc
                if not flags.values[g] and mflags.values[r]:
                    vals.valids[g] = mvals.valids[r]
                    if mvals.valids[r]:
                        vals.values[g] = mvals.values[r]
                    flags.values[g] = True
            elif not acc.valids[g] and macc.valids[r]:
                acc.values[g] = macc.values[r]; acc.valids[g] = True

    def final_merge(self, acc, idx) -> O.Col:
        return (acc[0] if isinstance(acc, tuple) else acc).to_col(idx)

    def final_type(self):
        return self.data_type


def make_agg(fexpr: E.AggFunctionExpr, input_schema: Schema) -> O.Agg:
    return FirstAgg(fexpr, input_schema) if fexpr.function in FIRST_FNS else O.Agg(fexpr, input_schema)


class AggExec(O.AggExec):
    """O.AggExec whose aggregates may include FIRST / FIRST_IGNORES_NULL"""

    def __init__(self, exec_mode, groupings, aggs, supports_partial_skipping, input_schema, batch_size: int = 10000):
        self.input_schema = input_schema
        self.groupings = list(groupings)
        self.agg_exprs = list(aggs)
        self.aggs = [make_agg(a.agg, input_schema) for a in aggs]
        self.modes = [a.mode for a in aggs]
        self.supports_partial_skipping = supports_partial_skipping
        self.batch_size = batch_size
        self.need_partial_update = any(m == E.PARTIAL for m in self.modes)
        self.need_partial_merge = any(m != E.PARTIAL for m in self.modes)
        self.need_final_merge = any(m == E.FINAL for m in self.modes)
        assert not (self.need_final_merge and any(m != E.FINAL for m in self.modes))
        gfields = [Field(g.field_name, g.expr.data_type(input_schema), g.expr.nullable(input_schema)) for g in groupings]
        if self.need_final_merge:
            afields = [Field(a.field_name, ag.final_type(), ag.nullable) for a, ag in zip(aggs, self.aggs)]
        else:
            afields = [Field(E.AGG_BUF_COLUMN_NAME, T.binary, False)]
        self.schema = Schema(gfields + afields)
        self.num_group_cols = len(gfields)


def brute_force_first(keys: list, values: list, ignore_nulls: bool) -> dict:
    """{key: value or None} straight from the definition: the first row of each key (the first row with a value when
    ignore_nulls).  `values` holds None for NULL."""
    out = {}
    for k, v in zip(keys, values):
        if k not in out:
            out[k] = v
        elif ignore_nulls and out[k] is None:
            out[k] = v
    return out


def freeze_first(dt: T.DataType, value, flag: bool = True) -> bytes:
    """the frozen bytes of one FIRST state (value None = NULL)"""
    acc = (O._PrimAcc(dt), _FlagAcc())
    for a in acc:
        a.resize(1)
    if value is not None:
        acc[0].values[0] = value; acc[0].valids[0] = True
    acc[1].values[0] = flag
    return acc[0].freeze(0) + acc[1].freeze(0)


def np_values(col: O.Col) -> list:
    return [None if not col.valid[i] else (col.values[i].item() if hasattr(col.values[i], "item") else col.values[i]) for i in range(len(col))]
