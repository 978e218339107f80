"""The fixed cost of an aggregation op around its update kernels: the table counters of every launch written into a pinned
snapshot by a kernel, streams and events recycled from one op to the next, and the hashed-slot emit skipped when the hashed
slots hold no group.  Every case is checked against the oracle."""
import threading

import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from oracle import blaze_oracle as O
from helpers import *

pytestmark = pytest.mark.gpu


def _sum_count_plans(keys):
    g = [E.GroupingExpr(c, E.Column(c)) for c in keys]
    aggs = [("s", E.AGG_SUM, "v"), ("c", E.AGG_COUNT, "v")]
    mk = lambda mode, src: [E.AggExpr(nm, mode, PL.create_agg(fn, [E.Column(col)] if mode == E.PARTIAL else [E.placeholder(T.int64)], src, T.int64))
                            for nm, fn, col in aggs]
    return g, mk


def _run(batches, keys, preds, conf):
    """Filter? -> AggExec(Partial) -> AggExec(Final) in one op on the GPU, and the same plan on the oracle"""
    leaf = PL.MemoryExec.from_arrow(batches, batches[0].schema)
    ins = leaf.schema()
    g, mk = _sum_count_plans(keys)
    partial = PL.AggExec(PL.HashAgg, g, mk(E.PARTIAL, ins), False, PL.FilterExec(preds, leaf) if preds else leaf)
    final = PL.AggExec(PL.HashAgg, g, mk(E.FINAL, partial.schema()), False, partial)
    got = PL.collect(final, conf)
    ob = oracle_batches(batches)
    op = O.AggExec(E.HASH_AGG, g, mk(E.PARTIAL, ins), False, ins)
    of = O.AggExec(E.HASH_AGG, g, mk(E.FINAL, op.schema), False, op.schema)
    exp = of.execute(op.execute(O.FilterExec(preds, ins).execute(ob) if preds else ob))
    assert_multiset_equal(got, exp)
    return final.last_metrics, sum(b.num_rows for b in got)


def _between(col, lo, hi):
    return [E.BinaryExpr(E.Column(col), "GtEq", E.Literal(lo, T.int64)), E.BinaryExpr(E.Column(col), "LtEq", E.Literal(hi, T.int64))]


@pytest.mark.parametrize("n, launch_rows", [(1_300_000, 1 << 16), (900_000, 150_000)])
def test_kernel_written_snapshots_under_deferral_and_growth(n, launch_rows):
    # one batch, cut into many launches; the keys are all distinct, so the hashed table hits its load limit while the next launch
    # is in flight and grows: the deferred rows of both launches are counted in the snapshots the kernel writes, then replayed
    rng = np.random.default_rng(n + launch_rows)
    k = rng.integers(0, 2**40, n, dtype=np.int64)
    v = rng.integers(-10**6, 10**6, n, dtype=np.int64)
    rb = pa.RecordBatch.from_arrays([pa.array(k), pa.array(v)], names=["k", "v"])
    conf = native.default_conf(agg_initial_groups=1024, staging_rows=0, max_launch_rows=launch_rows)
    m, groups = _run([rb], ["k"], [], conf)
    assert m["table_grow_count"] >= 1
    assert m["hot_kernel_launches"] >= (n + launch_rows - 1) // launch_rows
    assert m["num_groups"] == groups == len(np.unique(k))


def test_kernel_written_snapshots_dense_fused_filter():
    # the M2 shape (fused filter, two dense keys) over several launches per batch and several batches
    rng = np.random.default_rng(3)
    bs = []
    for _ in range(3):
        n = 400_000
        cols = [rng.integers(0, 1000, n), rng.integers(0, 1 << 10, n), rng.integers(0, 8, n), rng.integers(-10**6, 10**6, n)]
        bs.append(pa.RecordBatch.from_arrays([pa.array(c.astype(np.int64)) for c in cols], names=["f", "k1", "k2", "v"]))
    conf = native.default_conf(staging_rows=0, max_launch_rows=1 << 16, agg_initial_groups=1 << 13)
    m, groups = _run(bs, ["k1", "k2"], _between("f", 200, 399), conf)
    assert m["fast_path_launches"] >= 3 * 7
    assert m["num_groups"] == groups


def _dense_batches(rng, n, nb, outside):
    out = []
    for b in range(nb):
        k0 = rng.integers(0, 3000, n, dtype=np.int64)
        k1 = rng.integers(0, 8, n, dtype=np.int64)
        if b == 0:
            k0[:2], k1[:2] = [0, 2999], [0, 7]
        elif outside:                                 # keys outside the padded range sampled from the first batch: hashed slots
            k0[::101] += 100_000
        f = rng.integers(0, 100, n, dtype=np.int64)
        v = rng.integers(-10**6, 10**6, n, dtype=np.int64)
        out.append(pa.RecordBatch.from_arrays([pa.array(f), pa.array(k0), pa.array(k1), pa.array(v)], names=["f", "k0", "k1", "v"]))
    return out


@pytest.mark.parametrize("filtered", [False, True], ids=["no filter", "fused filter"])
@pytest.mark.parametrize("outside", [False, True], ids=["dense only", "later keys hashed"])
def test_hashed_emit_only_when_the_hashed_slots_hold_groups(outside, filtered):
    rng = np.random.default_rng(11 + 2 * outside + filtered)
    bs = _dense_batches(rng, 60_000, 3, outside)
    preds = _between("f", 20, 59) if filtered else []
    m, groups = _run(bs, ["k0", "k1"], preds, native.default_conf(staging_rows=0, agg_initial_groups=1024))
    assert m["fast_path_launches"] > 0
    assert m["num_groups"] == groups


def _device_to_numpy(d):
    import torch
    cols = []
    for i in range(d.array.n_children):
        c = d.array.children[i].contents
        if c.length == 0:
            cols.append(np.zeros(0, np.int64))
            continue

        class View:
            __cuda_array_interface__ = {"shape": (c.length * 8,), "typestr": "|u1", "data": (c.buffers[1], False), "version": 3}
        cols.append(torch.as_tensor(View(), device="cuda").view(torch.int64).cpu().numpy())
    return cols


def _check(cols, k, f, v):
    """cols: the pulled [k, SUM(v), COUNT(v)] of `f BETWEEN 200 AND 399` against numpy"""
    sel = (f >= 200) & (f <= 399)
    keys, inv = np.unique(k[sel], return_inverse=True)
    sums = np.zeros(len(keys), np.int64)
    np.add.at(sums, inv, v[sel])
    cnt = np.bincount(inv, minlength=len(keys))
    got_k, got_s, got_c = cols
    order = np.argsort(got_k)
    assert np.array_equal(got_k[order], keys)
    assert np.array_equal(got_s[order], sums)
    assert np.array_equal(got_c[order], cnt)


def test_recycled_streams_and_events_across_ops_and_threads():
    # many create / destroy cycles on two threads at once; each thread keeps the device array pulled from one op alive past
    # that op's destroy and across the ops after it (its memory is stream-ordered on the first op's stream), and reads it last
    import torch
    torch.cuda.init()
    ins = T.Schema([T.Field(n, T.int64, False) for n in ("f", "k", "v")])
    leaf = PL.MemoryExec(ins)
    g, mk = _sum_count_plans(["k"])
    partial = PL.AggExec(PL.HashAgg, g, mk(E.PARTIAL, ins), False, PL.FilterExec(_between("f", 200, 399), leaf))
    plan = PL.AggExec(PL.HashAgg, g, mk(E.FINAL, partial.schema()), False, partial).plan_bytes()
    errors = []

    def worker(t):
        try:
            rng = np.random.default_rng(100 + t)
            kept = None
            for i in range(40):
                n = int(rng.integers(1, 20_000))
                f, k, v = rng.integers(0, 1000, n), rng.integers(0, 50 + 500 * (i % 3), n), rng.integers(-10**6, 10**6, n)
                rb = pa.RecordBatch.from_arrays([pa.array(x.astype(np.int64)) for x in (f, k, v)], names=["f", "k", "v"])
                with native.NativeOp(plan, native.default_conf(staging_rows=0), 0) as op:
                    op.push(rb)
                    op.finish()
                    d = op.pull_device()
                    assert op.pull_device() is None
                if d is None:
                    assert not ((f >= 200) & (f <= 399)).any()
                    continue
                if kept is None and i >= 5:
                    kept = (d, f, k, v)                 # kept past its op's destroy and the ops after it
                    continue
                _check(_device_to_numpy(d), k, f, v)
                native.release_device_array(d)
            d, f, k, v = kept
            _check(_device_to_numpy(d), k, f, v)
            native.release_device_array(d)
        except BaseException as e:                      # reported by the main thread
            errors.append(e)
    ts = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0]
