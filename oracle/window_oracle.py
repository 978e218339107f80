"""WindowExec restated row by row on the numpy oracle of oracle/blaze_oracle.py: the three processors of the reference
(datafusion-ext-plans/src/window/processors/{row_number,rank,agg}_processor.rs) with their state carried from one batch to the
next, the group limit and output assembly of window_exec.rs:203-266, and the Window-over-WindowGroupLimit combining rule
(window_exec.rs:166-185)."""
from typing import List, Optional, Sequence

import numpy as np

from blaze_b200 import exprs as E
from blaze_b200 import types as T
from blaze_b200.types import Field, Schema

from .blaze_oracle import Agg, Batch, Col, OracleError, cast, evaluate


def wrap_i32(v: int) -> int:
    return (int(v) + (1 << 31)) % (1 << 32) - (1 << 31)


def key_rows(cols: Sequence[Col], n: int) -> List[tuple]:
    """the arrow-row encoding's equality: NULL equals NULL and differs from every value; values are equal iff their bits are
    (floats by their IEEE bits, so -0.0 != +0.0 and NaNs only equal with the same payload).  No key column: every row is ()."""
    out = []
    for r in range(n):
        row = []
        for c in cols:
            if not c.valid[r]:
                row.append(("null",))
            elif c.dtype.id in (T.FLOAT32, T.FLOAT64):
                row.append(("v", np.asarray(c.values[r]).tobytes()))
            else:
                row.append(("v", int(c.values[r])))
        out.append(tuple(row))
    return out


class WindowExec:
    """WindowContext::try_new + execute_window.  order_spec = [(expr, descending, nulls_first)]: the sort options never take part
    in equality."""

    def __init__(self, window_exprs: Sequence[E.WindowExpr], partition_spec: Sequence[E.Expr], order_spec, input_schema: Schema,
                 group_limit: Optional[int] = None, output_window_cols: bool = True):
        self.window_exprs, self.partition_spec = list(window_exprs), list(partition_spec)
        self.order_spec = [e for e, _d, _nf in order_spec]
        self.input_schema, self.group_limit, self.output_window_cols = input_schema, group_limit, output_window_cols
        if group_limit is not None and len(self.window_exprs) != 1:
            raise OracleError("a group limit needs exactly one window expression")          # window_exec.rs:228
        self.schema = Schema(list(input_schema) + ([w.field for w in self.window_exprs] if output_window_cols else []))
        self.aggs = [Agg(E.AggFunctionExpr(w.agg_func, w.children, w.return_type), input_schema) if w.func_type == E.WINDOW_AGG else None
                     for w in self.window_exprs]

    @staticmethod
    def combine(parent: "WindowExec", child: "WindowExec") -> "WindowExec":
        """a WindowExec without a limit over one with a limit: the parent's expressions, the child's limit, output_window_cols
        = true, over the child's input"""
        if parent.group_limit is not None or child.group_limit is None:
            raise OracleError("only a WindowExec without a limit combines with a group-limited child")
        w = WindowExec([], parent.partition_spec, [(e, False, False) for e in parent.order_spec], child.schema, None, True)
        w.window_exprs, w.aggs, w.group_limit = parent.window_exprs, parent.aggs, child.group_limit
        w.input_schema = child.input_schema
        w.schema = Schema(list(child.input_schema) + [x.field for x in parent.window_exprs])
        return w

    def _window_column(self, k: int, st: dict, batch: Batch, prow, orow) -> Col:
        w, n = self.window_exprs[k], batch.num_rows
        has_partition = bool(self.partition_spec)
        if w.func_type == E.WINDOW_FUNC:
            vals = np.zeros(n, np.int32)
            for r in range(n):
                same = not has_partition or prow[r] == st["partition"]
                if not same:
                    st["partition"] = prow[r]
                if w.window_func == E.ROW_NUMBER:                       # row_number_processor.rs
                    st["rn"] = wrap_i32((0 if not same else st["rn"]) + 1)
                    vals[r] = st["rn"]
                    continue
                if same:                                                # rank_processor.rs
                    if orow[r] == st["order"]:
                        st["equals"] = wrap_i32(st["equals"] + 1)
                    else:
                        st["rank"] = wrap_i32(st["rank"] + (1 if w.window_func == E.DENSE_RANK else st["equals"]))
                        st["equals"], st["order"] = 1, orow[r]
                else:
                    st["rank"], st["equals"], st["order"] = 1, 1, orow[r]
                vals[r] = st["rank"]
            return Col(T.int32, vals, np.ones(n, bool))
        agg = self.aggs[k]                                              # agg_processor.rs
        args = [evaluate(e, batch).broadcast(n) for e in agg.exprs]
        outs = []
        for r in range(n):
            same = not has_partition or prow[r] == st["partition"]
            if not same:
                st["partition"] = prow[r]
            if not same or st["acc"] is None:
                st["acc"] = agg.create_acc()
                Agg.acc_resize(st["acc"], 1)
            agg.partial_update(st["acc"], [0], args, [r])
            outs.append(agg.final_merge(st["acc"], [0]))
        dt = outs[0].dtype
        valid = np.array([bool(c.valid[0]) for c in outs], bool)
        if dt.id == T.DECIMAL128:
            vals = np.empty(n, object)
            vals[:] = [c.values[0] for c in outs]
        else:
            vals = np.array([c.values[0] for c in outs], dtype=outs[0].values.dtype)
        return Col(dt, vals, valid)

    def execute(self, batches: Sequence[Batch]) -> List[Batch]:
        states = [{"partition": (), "order": (), "rn": 0, "rank": 0, "equals": 1, "acc": None} for _ in self.window_exprs]
        out = []
        for b in batches:
            n = b.num_rows
            if n == 0:
                continue
            prow = key_rows([evaluate(e, b).broadcast(n) for e in self.partition_spec], n)
            orow = key_rows([evaluate(e, b).broadcast(n) for e in self.order_spec], n)
            wcols = [self._window_column(k, states[k], b, prow, orow) for k in range(len(self.window_exprs))]
            cols = list(b.cols)
            if self.group_limit is not None:                            # window_exec.rs:227-235: the limit as i32
                keep = np.nonzero(wcols[0].values.astype(np.int64) <= wrap_i32(self.group_limit))[0]
                cols = [c.take(keep) for c in cols]
                wcols = [c.take(keep) for c in wcols]
                n = len(keep)
            if self.output_window_cols:
                cols += wcols
            cols = [c if c.dtype == f.dtype else cast(c, f.dtype) for c, f in zip(cols, self.schema)]
            if n:
                out.append(Batch(self.schema, cols, n))
        return out
