"""The WindowExec oracle (oracle/window_oracle.py) pinned by the reference's goldens (tests/golden/window_kats.json), checked against
an independent brute-force restatement (each row rescanned from its partition start), and for its state across batches, the group
limit's `as i32` and the combining rule."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, types as T
from oracle import blaze_oracle as O
from oracle import window_oracle as W
from helpers import split_batches, with_nulls
from window_cases import KATS, brute_force, kat_input, kat_window, oracle_run, sorted_table, window_expr


@pytest.mark.parametrize("batch_rows", [None, 1, 3])
@pytest.mark.parametrize("case", KATS, ids=[c["name"] for c in KATS])
def test_kats(case, batch_rows):
    schema, rb = kat_input(case)
    exprs, part, order = kat_window(case, schema)
    batches = [rb] if batch_rows is None else split_batches(rb, batch_rows)
    osch, out = oracle_run(schema, exprs, part, order, batches, case["group_limit"], case["output_window_cols"])
    t = pa.Table.from_batches([O.batch_to_arrow(b) for b in out])
    for name, vals in case["expected"].items():
        assert t.column(name).to_pylist() == vals, name


def _table(n, seed, key_dtype=np.int64, domain=4):
    rng = np.random.default_rng(seed)
    cols = [with_nulls(rng, rng.integers(0, domain, n).astype(key_dtype), 0.2) for _ in range(2)]
    cols.append(with_nulls(rng, rng.integers(-50, 50, n).astype(np.int64), 0.3))
    return sorted_table(pa.RecordBatch.from_arrays(cols, names=["p", "o", "v"]), ["p", "o"])


@pytest.mark.parametrize("part,order", [(["p"], ["o"]), ([], ["o"]), (["p"], []), ([], []), (["p", "o"], [])])
@pytest.mark.parametrize("fn,arg", [("row_number", None), ("rank", None), ("dense_rank", None), ("sum", "v"), ("count", "v"), ("min", "v"), ("max", "v")])
def test_oracle_matches_brute_force(part, order, fn, arg):
    rb = _table(400, seed=len(part) * 10 + len(order))
    schema = T.from_arrow_schema(rb.schema)
    exprs = [window_expr("w", fn, arg, schema)]
    _, out = oracle_run(schema, exprs, [E.Column(c) for c in part], [(E.Column(c), False, True) for c in order], split_batches(rb, 37))
    got = pa.Table.from_batches([O.batch_to_arrow(b) for b in out]).column("w").to_pylist()
    assert got == brute_force(rb, fn, part, order, arg)


def test_float_key_equality_is_bitwise():
    v = np.array([0.0, -0.0, -0.0, np.nan, np.nan, 1.0], np.float64)
    rb = pa.RecordBatch.from_arrays([pa.array(v), pa.array([None, None, 1.0, 1.0, 2.0, 2.0])], names=["k", "x"])
    schema = T.from_arrow_schema(rb.schema)
    _, out = oracle_run(schema, [window_expr("rn", "row_number")], [E.Column("k")], [], [rb])
    assert O.batch_to_arrow(out[0]).column(2).to_pylist() == [1, 1, 2, 1, 2, 1]
    _, out = oracle_run(schema, [window_expr("rk", "rank")], [], [(E.Column("x"), False, True)], [rb])
    assert O.batch_to_arrow(out[0]).column(2).to_pylist() == [1, 1, 3, 3, 5, 5]        # NULL == NULL, NULL != 1.0


@pytest.mark.parametrize("k,kept", [(0, 0), (1, 3), (2**31, 0), (2**32 - 1, 0), (2**32 + 1, 3)])
def test_group_limit_is_compared_as_i32(k, kept):
    rb = _table(60, seed=2, domain=3)
    schema = T.from_arrow_schema(rb.schema)
    _, out = oracle_run(schema, [window_expr("rn", "row_number")], [E.Column("p")], [(E.Column("o"), False, True)], [rb], k % 2**32 if k < 2**32 else k, False)
    n = sum(b.num_rows for b in out)
    npart = len(set(rb.column(0).to_pylist()))
    assert n == (kept // 3) * npart if kept else n == 0


def test_combining_rule():
    rb = _table(200, seed=4)
    schema = T.from_arrow_schema(rb.schema)
    part, order = [E.Column("p")], [(E.Column("o"), False, True)]
    child = W.WindowExec([window_expr("w", "rank")], part, order, schema, 2, False)
    parent = W.WindowExec([window_expr("rn", "row_number"), window_expr("s", "sum", "v", schema)], part, order, child.schema)
    comb = W.WindowExec.combine(parent, child)
    out = pa.Table.from_batches([O.batch_to_arrow(b) for b in comb.execute([O.batch_from_arrow(b) for b in split_batches(rb, 50)])])
    assert out.column_names == ["p", "o", "v", "rn", "s"]
    assert max(out.column("rn").to_pylist()) <= 2                 # the parent's row_number limited by the child's k (rn <= 2)
    with pytest.raises(O.OracleError):
        W.WindowExec.combine(child, parent)
