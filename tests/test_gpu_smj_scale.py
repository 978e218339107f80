"""SortMergeJoinExec at scale: 2^24 left rows against 2^22 right rows with uniform keys, with Zipf(1.1)-skewed left keys (hot key runs
that span many left batches), and the two-key MJ1 shape of tools/bench_shapes.py — every join type, against tests/vector_ref.py,
plus the output order each join type promises (tests/test_gpu_smj.py::check_order)."""
import numpy as np
import pyarrow as pa
import pytest

import vector_ref as V
from blaze_b200 import native, plans as PL
from helpers import split_batches
from test_gpu_smj import ALL_JT, JT_NAME, check_order, run, sorted_pos

pytestmark = pytest.mark.gpu

NL, NR = 1 << 24, 1 << 22
CONF = native.default_conf(staging_rows=0)
_CACHE = {}


def _sorted_batch(keys, valid, payload, tag):
    """rows sorted ascending by the keys (NULLs first), with row ids of that order"""
    kcols = [np.where(valid, k, 0) for k in keys]
    perm = np.lexsort(kcols[::-1] + [valid.astype(np.int8)])                  # NULL keys (valid 0) first, then the keys
    n = len(valid)
    cols = [pa.array(k[perm], mask=~valid[perm]) for k in keys]
    cols += [pa.array(np.arange(n, dtype=np.int64)), pa.array(payload[perm])]
    names = [f"k{i}{tag}" for i in range(len(keys))] + [f"id{tag}", f"v{tag}"]
    return pa.RecordBatch.from_arrays(cols, names=names)


def shape(name):
    if name in _CACHE:
        return _CACHE[name]
    rng = np.random.default_rng({"uniform": 1, "zipf": 2, "mj1": 3}[name])
    if name == "uniform":
        lk, rk = [rng.integers(0, 1 << 23, NL)], [rng.integers(0, 1 << 23, NR)]
    elif name == "zipf":
        lk = [(rng.zipf(1.1, NL) % (1 << 22)).astype(np.int64)]
        rk = [rng.permutation(1 << 23)[:NR].astype(np.int64)]                  # unique right keys: the output stays near 2^24 rows
    else:                                                                       # store_sales ⋈ store_returns on (item_sk, ticket): ~10 % of the left rows match
        item, ticket = rng.integers(0, 1 << 18, NL), rng.integers(0, 1 << 30, NL)
        pick = rng.choice(NL, NR, replace=False)
        ri, rt = item[pick].copy(), ticket[pick].copy()
        fresh = rng.random(NR) < 0.6                                           # returns whose sale is not on this side
        rt[fresh] = rng.integers(1 << 30, 1 << 31, int(fresh.sum()))
        lk, rk = [item, ticket], [ri, rt]
    lv, rv = rng.random(NL) >= 0.01, rng.random(NR) >= 0.01
    lrb = _sorted_batch(lk, lv, rng.integers(-10**9, 10**9, NL), "l")
    rrb = _sorted_batch(rk, rv, rng.integers(-10**9, 10**9, NR), "r")
    lcols, rcols = V.from_batches([lrb]), V.from_batches([rrb])
    opts = [(True, True)] * len(lk)
    _CACHE[name] = (lrb, rrb, len(lk), lcols, rcols, sorted_pos(lrb, len(lk), opts), sorted_pos(rrb, len(lk), opts))
    return _CACHE[name]


@pytest.mark.parametrize("jt", ALL_JT, ids=lambda j: JT_NAME[j])
@pytest.mark.parametrize("name", ["uniform", "zipf", "mj1"])
def test_scale(name, jt):
    lrb, rrb, nkeys, lcols, rcols, lsorted, rsorted = shape(name)
    opts = [(True, True)] * nkeys
    on = [(f"k{k}l", f"k{k}r") for k in range(nkeys)]
    _, out = run(split_batches(lrb, 1 << 22), split_batches(rrb, 1 << 21), on, jt, opts, CONF, sort_left=False, sort_right=False)
    got = V.from_batches(out)
    exp = V.join(lcols, rcols, [(k, k) for k in range(nkeys)], jt, V.RIGHT_SIDE)
    ids = [nkeys] if jt in (PL.JOIN_SEMI, PL.JOIN_ANTI, PL.JOIN_EXISTENCE) else [nkeys, lrb.num_columns + nkeys]   # row ids make every row unique
    V.assert_same_rows(got, exp, by=ids)
    check_order(got, jt, nkeys, lrb, rrb, opts, lsorted, rsorted)
