"""Entry order of a two-key dense table: the key with the shorter padded span indexes the table's rows, so that the
margins of a short key do not interleave dead entries with live ones (M2's k2 has 8 values and a span of 20).  Each case
runs with and without a fused filter (tile kernel / row kernels), over several batches whose later rows hold keys outside
the range sampled from the first batch (hashed slots), and is checked against the oracle."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, plans as PL, types as T, native
from oracle import blaze_oracle as O
from helpers import *

pytestmark = pytest.mark.gpu


def _batches(rng, n, r0, r1, nb):
    out = []
    for b in range(nb):
        k0 = rng.integers(0, r0, n, dtype=np.int64)
        k1 = rng.integers(0, r1, n, dtype=np.int64)
        if b == 0:
            k0[:2], k1[:2] = [0, r0 - 1], [0, r1 - 1]
        else:                                         # keys outside the padded range of the first batch: hashed slots
            k0[::97] += 3 * r0
            k1[::89] -= 3 * r1
        f = rng.integers(0, 100, n, dtype=np.int64)
        v = rng.integers(-10**6, 10**6, n, dtype=np.int64)
        out.append(pa.RecordBatch.from_arrays([pa.array(f), pa.array(k0), pa.array(k1), pa.array(v)], names=["f", "k0", "k1", "v"]))
    return out


@pytest.mark.parametrize("r0, r1", [(5000, 8), (8, 5000), (300, 300)], ids=["key1 shorter", "key0 shorter", "equal"])
@pytest.mark.parametrize("filtered", [False, True], ids=["no filter", "fused filter"])
def test_two_key_dense_layout(r0, r1, filtered):
    rng = np.random.default_rng(r0 * 7 + r1 + filtered)
    bs = _batches(rng, 50_000, r0, r1, 3)
    leaf = PL.MemoryExec.from_arrow(bs, bs[0].schema)
    ins = leaf.schema()
    preds = [E.BinaryExpr(E.Column("f"), "GtEq", E.Literal(20, T.int64)), E.BinaryExpr(E.Column("f"), "LtEq", E.Literal(39, T.int64))] if filtered else []
    g = [E.GroupingExpr(c, E.Column(c)) for c in ("k0", "k1")]
    aggs = [("s", E.AGG_SUM, "v"), ("c", E.AGG_COUNT, "v")]
    mk = lambda mode, src: [E.AggExpr(nm, mode, PL.create_agg(fn, [E.Column(col)] if mode == E.PARTIAL else [E.placeholder(T.int64)], src, T.int64))
                            for nm, fn, col in aggs]
    partial = PL.AggExec(PL.HashAgg, g, mk(E.PARTIAL, ins), False, PL.FilterExec(preds, leaf) if preds else leaf)
    final = PL.AggExec(PL.HashAgg, g, mk(E.FINAL, partial.schema()), False, partial)
    got = PL.collect(final, native.default_conf(staging_rows=0, agg_initial_groups=1024))
    assert final.last_metrics["fast_path_launches"] > 0
    ob = oracle_batches(bs)
    op = O.AggExec(E.HASH_AGG, g, mk(E.PARTIAL, ins), False, ins)
    of = O.AggExec(E.HASH_AGG, g, mk(E.FINAL, op.schema), False, op.schema)
    assert_multiset_equal(got, of.execute(op.execute(O.FilterExec(preds, ins).execute(ob) if preds else ob)))
