"""The exact aggregate reference (tests/exact_agg.py) against the oracle, on every numeric-edge family: equal bits wherever
the result does not depend on the summation order (the -0.0 sums included, which confirms the reference's
store-the-first-value-then-add semantics), the oracle's sequential f64 sums inside the proven interval elsewhere, and the
IEEE totalOrder key model against a hand-ordered list."""
import math

import numpy as np
import pytest

from blaze_b200 import exprs as E, plans as PL
from oracle import blaze_oracle as O
import exact_agg as X


def _oracle_groups(tab, specs):
    ins = PL.MemoryExec.from_arrow(tab.batches, tab.schema).schema()
    g = [E.GroupingExpr("k", E.Column("k"))]
    mk = lambda mode, sch: [E.AggExpr(nm, mode, PL.create_agg(fn, [E.Column(c) if c else E.Literal(1, X.T.int64)] if mode == E.PARTIAL
                                                                   else [E.placeholder(ins[ins.index_of(c)].dtype if c else X.T.int64)], sch, rt))
                            for nm, fn, c, rt in specs]
    op = O.AggExec(E.HASH_AGG, g, mk(E.PARTIAL, ins), False, ins)
    of = O.AggExec(E.HASH_AGG, g, mk(E.FINAL, ins), False, op.schema)
    out = {}
    for b in of.execute(op.execute([O.batch_from_arrow(rb) for rb in tab.batches])):
        for r in range(b.num_rows):
            vals = [None if not c.valid[r] else (np.float32(c.values[r]) if c.dtype.id == X.T.FLOAT32 else float(c.values[r]) if c.dtype.is_float else int(c.values[r]))
                    for c in b.cols]
            out[(vals[0],)] = vals[1:]
    return out


def _order_dependent_in_the_oracle(vals):
    """MIN / MAX groups where Rust's partial_cmp depends on the row order: a NaN, or both zeros"""
    v = [x for x in vals if x is not None]
    return any(x != x for x in v) or (any(x == 0 and math.copysign(1, x) < 0 for x in v) and any(x == 0 and math.copysign(1, x) > 0 for x in v))


@pytest.mark.parametrize("shape", list(X.SHAPES))
def test_reference_agrees_with_the_oracle(shape):
    sh = X.SHAPES[shape]
    tab = X.family(sh.family)
    specs = sh.specs
    exp = X.expected_groups([(k,) for k in tab.keys], tab.cols, specs, tab.types)
    got = _oracle_groups(tab, specs)
    assert got.keys() == exp.keys()
    rows = {}
    for r, k in enumerate(tab.keys):
        rows.setdefault(k, []).append(r)
    checked = {"exact": 0, "interval": 0, "order-dependent": 0}
    for k, ev in exp.items():
        for (nm, fn, col, _), e, g in zip(specs, ev, got[k]):
            if fn in (E.AGG_MIN, E.AGG_MAX) and col and tab.types[col].is_float and _order_dependent_in_the_oracle([tab.cols[col][r] for r in rows[k[0]]]):
                checked["order-dependent"] += 1                          # the documented deviation: totalOrder on the GPU
                continue
            assert X.matches(e, g), f"group {k} ({tab.kinds.get(k[0])}) {nm}: reference {e!r}, oracle {g!r}"
            checked["interval" if isinstance(e, X.Interval) else "exact"] += 1
    assert checked["exact"] > 0


def test_negative_zero_sums_are_negative_zero_in_the_oracle():
    tab = X.family("f64")
    specs = X.SHAPES["f64 sum avg count"].specs
    got = _oracle_groups(tab, specs)
    neg = [k for k, kind in tab.kinds.items() if kind in ("neg_zero", "neg_zero_nulls")]
    assert len(neg) > 20
    for k in neg:
        s, a, _ = got[(k,)]
        assert str(s) == "-0.0" and str(a) == "-0.0", f"group {k}: {s}, {a}"


def test_order_free_sums_are_exact_and_the_rest_intervals():
    assert X.f64_sum([-0.0, -0.0]) == 0 and str(X.f64_sum([-0.0, -0.0])) == "-0.0"
    assert str(X.f64_sum([-0.0, 0.0])) == "0.0" and str(X.f64_sum([1.0, -1.0, -0.0])) == "0.0"
    assert X.f64_sum([1.5e308] * 3) == math.inf and X.f64_sum([-1.5e308] * 3) == -math.inf
    assert math.isnan(X.f64_sum([math.inf, -math.inf])) and math.isnan(X.f64_sum([1.0, math.nan]))
    assert X.f64_sum([2.0 ** 40, 0.25, -(2.0 ** 40)]) == 0.25                   # the small row survives in any order
    assert X.f64_sum([5e-324, 5e-324, -1e-323 * 3]) == -2e-323
    iv = X.f64_sum([1e16, 1.0, -1e16])
    assert isinstance(iv, X.Interval) and iv.center == 1 and 0.0 in iv and 1.0 in iv and 6.0 not in iv
    assert str(X.f64_avg([-0.0, -0.0, -0.0])) == "-0.0"
    assert X.dec_avg([-7, 0], X.D38_0, X.D38_0) == -4                           # div_euclid rounds toward -inf
    assert X.dec_sum([10 ** 38 - 1] * 2, X.D38_0, X.D38_0) == X.wrap(2 * (10 ** 38 - 1), 128)
    assert X.dec_avg([10 ** 34, 5], X.D38_2, X.T.decimal128(38, 6)) == 50000    # the cast of 10^34 overflows: NULL, not counted


def test_total_order_key_model():
    ordered64 = [X.NEG_NAN, -math.inf, -X.DBL_MAX, -2.0, -X.DBL_MIN, -5e-324, -0.0, 0.0, 5e-324, X.DBL_MIN, 1.5, X.DBL_MAX, math.inf, math.nan]
    keys = [X.total_order_key(X.f64_bits(x), 64) for x in ordered64]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    ordered32 = [X.to_f32(x) for x in [X.NEG_NAN, -math.inf, -X.F32_MAX, -2.0, -1e-45, -0.0, 0.0, 1e-45, 1.5, X.F32_MAX, math.inf, math.nan]]
    keys = [X.total_order_key(X.f32_bits(x), 32) for x in ordered32]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    assert X.f32_bits(ordered32[0]) >> 31 == 1
    assert str(X.float_minmax([0.0, -0.0], E.AGG_MIN, 64)) == "-0.0" and str(X.float_minmax([-0.0, 0.0], E.AGG_MAX, 64)) == "0.0"
    assert math.copysign(1, X.float_minmax([1.0, X.NEG_NAN], E.AGG_MIN, 64)) < 0 and X.float_minmax([1.0, X.NEG_NAN], E.AGG_MAX, 64) == 1.0
