"""ExpandExec restated on the numpy oracle of oracle/blaze_oracle.py (expressions, casts, batches)."""
from typing import List, Sequence

from blaze_b200 import exprs as E
from blaze_b200.types import Schema

from .blaze_oracle import Batch, Col, OracleError, cast, evaluate


class ExpandExec:
    """datafusion-ext-plans/src/expand_exec.rs: try_new (:49-77) checks that every projection has an expression of the
    field's type for every schema field; execute_expand (:147-187) evaluates each projection in turn over every input batch
    and sends it as its own batch (expressions zipped with the fields: extra ones are ignored; a differing type is cast)."""

    def __init__(self, schema: Schema, projections: Sequence[Sequence[E.Expr]], input_schema: Schema):
        for proj in projections:
            for i, f in enumerate(schema):
                got = proj[i].data_type(input_schema) if i < len(proj) else None
                if got != f.dtype:
                    raise OracleError(f"ExpandExec data type not matches: {got} vs {f.dtype}")
        self.schema = schema
        self.projections = [list(p) for p in projections]

    def execute(self, batches: Sequence[Batch]) -> List[Batch]:
        out = []
        for b in batches:
            if b.num_rows == 0:                     # sender.send drops empty batches (execution_context.rs:713-716)
                continue
            for proj in self.projections:
                cols = []
                for e, f in zip(proj, self.schema):
                    c = evaluate(e, b).broadcast(b.num_rows)
                    if c.dtype != f.dtype:
                        c = cast(c, f.dtype)
                    cols.append(Col(c.dtype, c.values, c.valid))
                out.append(Batch(self.schema, cols, b.num_rows))
        return out
