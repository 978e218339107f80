"""SortMergeJoinExec on the GPU through the C ABI: the reference's join goldens with both sides through SortExec, every
asc x nulls_first combination over NULL keys of every key type, left batches whose key runs straddle batch boundaries, a right op
that emits several batches, output chunks, edge inputs, unsorted input, misuse of the ABI, and a fused
SortExec -> SMJ -> Project -> AggExec op — against tests/vector_ref.py and the oracle, plus a vectorised check of the output
order each join type promises (DESIGN.md §3.14)."""
import numpy as np
import pyarrow as pa
import pytest

import vector_ref as V
from blaze_b200 import exprs as E, native, plans as PL, types as T
from helpers import split_batches, with_nulls
from join_goldens import CASES, arrow_batches
from oracle import blaze_oracle as O
from oracle import join_oracle as J

pytestmark = pytest.mark.gpu

WIRE = {J.INNER: PL.JOIN_INNER, J.LEFT: PL.JOIN_LEFT, J.RIGHT: PL.JOIN_RIGHT, J.FULL: PL.JOIN_FULL, J.LEFT_SEMI: PL.JOIN_SEMI, J.LEFT_ANTI: PL.JOIN_ANTI, J.EXISTENCE: PL.JOIN_EXISTENCE}
ALL_JT = [PL.JOIN_INNER, PL.JOIN_LEFT, PL.JOIN_RIGHT, PL.JOIN_FULL, PL.JOIN_SEMI, PL.JOIN_ANTI, PL.JOIN_EXISTENCE]
JT_NAME = {PL.JOIN_INNER: "inner", PL.JOIN_LEFT: "left", PL.JOIN_RIGHT: "right", PL.JOIN_FULL: "full", PL.JOIN_SEMI: "semi", PL.JOIN_ANTI: "anti", PL.JOIN_EXISTENCE: "existence"}
NOSTAGE = native.default_conf(staging_rows=0)


def _plan(lb, rb, on, jt, opts, sort_left=True, sort_right=True, lschema=None, rschema=None):
    left = PL.MemoryExec.from_arrow(lb, lschema or lb[0].schema)
    right = PL.MemoryExec.from_arrow(rb, rschema or rb[0].schema)
    ls, rs = left.schema(), right.schema()
    if sort_left:
        left = PL.SortExec(left, [(E.Column(l), not a, nf) for (l, _), (a, nf) in zip(on, opts)])
    if sort_right:
        right = PL.SortExec(right, [(E.Column(r), not a, nf) for (_, r), (a, nf) in zip(on, opts)])
    return PL.SortMergeJoinExec(PL.build_join_schema(ls, rs, jt), left, right, [(E.Column(l), E.Column(r)) for l, r in on], opts, jt)


def run(lb, rb, on, jt, opts, conf=None, **kw):
    plan = _plan(lb, rb, on, jt, opts, **kw)
    return plan, PL.collect(plan, conf)


# ---- goldens ---------------------------------------------------------------------------------------------------------------
def _key(t):
    return tuple((x is None, x if x is not None else 0) for x in t)


def _rows(batches):
    rows = []
    for b in [O.batch_from_arrow(x) for x in batches]:
        for r in range(b.num_rows):
            rows.append(tuple(None if not c.valid[r] else (c.values[r].item() if hasattr(c.values[r], "item") else c.values[r]) for c in b.cols))
    return sorted(rows, key=_key)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_reference_join_goldens(case):
    name, left, right, on, jt, expected = case[:6]
    dtype = case[6] if len(case) > 6 else "int32"
    lb, rb = arrow_batches(left, dtype), arrow_batches(right, dtype)
    plan, out = run(lb, rb, on, WIRE[jt], [(True, True)] * len(on))
    got = _rows(out)
    if dtype != "int32":
        got = [tuple(None if x is None else int(x) for x in r) for r in got]
    assert got == sorted(expected, key=_key)
    assert plan.last_metrics["gpu_kernel_launches"] > 0


# ---- random inputs against vector_ref, with the ordering contract ------------------------------------------------------------
KEY_TYPES = {"i32": (pa.int32(), np.int32), "i64": (pa.int64(), np.int64), "date32": (pa.date32(), np.int32), "ts": (pa.timestamp("us"), np.int64)}


def side(rng, n, tag, ktype, nkeys, krange, null_frac):
    pt, nt = KEY_TYPES[ktype]
    cols, names = [], []
    for k in range(nkeys):
        v = rng.integers(-krange, krange, n).astype(nt)
        cols.append(with_nulls(rng, v, null_frac, pa.int32() if nt == np.int32 else pa.int64()).cast(pt))
        names.append(f"k{k}{tag}")
    cols.append(pa.array(np.arange(n, dtype=np.int64)))                                           # row id in input order
    names.append(f"id{tag}")
    cols.append(with_nulls(rng, rng.integers(-10**9, 10**9, n, dtype=np.int64), 0.1))
    names.append(f"v{tag}")
    cols.append(pa.array(rng.integers(-100, 100, n).astype(np.int16), pa.int16()))
    names.append(f"s{tag}")
    return pa.RecordBatch.from_arrays(cols, names=names)


def sorted_pos(rb, nkeys, opts):
    """position of every input row in the stably sorted input, and the rank of its key group there"""
    cols = V.from_batches([rb])
    perm = V.sort_permutation(cols, [(k, not a, nf) for k, (a, nf) in enumerate(opts[:nkeys])])
    pos = np.empty(len(perm), np.int64)
    pos[perm] = np.arange(len(perm))
    keys = [c.take(perm) for c in cols[:nkeys]]
    new = np.ones(len(perm), bool)
    if len(perm) > 1:
        same = np.ones(len(perm) - 1, bool)
        for c in keys:
            same &= (c.valid[1:] == c.valid[:-1]) & (c.values[1:] == c.values[:-1])
        new[1:] = ~same
    grp = np.cumsum(new) - 1
    return pos, grp[pos]


def check_order(got, jt, nkeys, lrb, rrb, opts, lsorted=None, rsorted=None):
    """the row order the join type promises (got: VCols of the output; l/rsorted: sorted_pos of a side, when already known)"""
    nl = lrb.num_columns
    lid, rid = got[nkeys], (got[nl + nkeys] if jt not in (PL.JOIN_SEMI, PL.JOIN_ANTI, PL.JOIN_EXISTENCE) else None)
    if jt == PL.JOIN_FULL:
        return
    if jt == PL.JOIN_RIGHT:
        rpos, rgrp = rsorted or sorted_pos(rrb, nkeys, opts)
        g = rgrp[rid.values]
        assert np.all(np.diff(g) >= 0), "Right: rows do not follow the right keys' order"
        same = g[1:] == g[:-1]
        assert not np.any(same & ~lid.valid[:-1] & lid.valid[1:]), "Right: a right-only row before a left-driven row of its key"
        return
    lpos, _ = lsorted or sorted_pos(lrb, nkeys, opts)
    p = lpos[lid.values]
    assert lid.valid.all()
    assert np.all(np.diff(p) >= 0), "rows do not follow the left input order"
    if rid is not None and len(p) > 1 and rrb.num_rows:
        rpos, _ = rsorted or sorted_pos(rrb, nkeys, opts)
        same = (p[1:] == p[:-1]) & rid.valid[1:] & rid.valid[:-1]
        r = rpos[rid.values]
        assert np.all(r[1:][same] > r[:-1][same]), "matches of a left row not in right input order"


def compare(out, lrb, rrb, nkeys, jt, opts):
    got = V.from_batches(out, ncols=None) if out else None
    on = [(k, k) for k in range(nkeys)]
    exp = V.join(V.from_batches([lrb]), V.from_batches([rrb]), on, jt, V.RIGHT_SIDE)
    if got is None:
        assert len(exp[0]) == 0
        return
    V.assert_same_rows(got, exp)
    check_order(got, jt, nkeys, lrb, rrb, opts)


@pytest.mark.parametrize("jt", ALL_JT, ids=lambda j: JT_NAME[j])
@pytest.mark.parametrize("ktype", list(KEY_TYPES))
@pytest.mark.parametrize("nkeys", [1, 2])
@pytest.mark.parametrize("asc,nf", [(True, True), (True, False), (False, True), (False, False)], ids=["asc_nf", "asc_nl", "desc_nf", "desc_nl"])
def test_sort_options_null_keys_and_key_types(jt, ktype, nkeys, asc, nf):
    rng = np.random.default_rng(1000 * jt + 100 * list(KEY_TYPES).index(ktype) + 10 * nkeys + 2 * asc + nf)
    krange = 40 if nkeys == 1 else 6
    lrb, rrb = side(rng, 3_000, "l", ktype, nkeys, krange, 0.08), side(rng, 1_200, "r", ktype, nkeys, krange, 0.08)
    opts = [(asc, nf)] * nkeys
    if nkeys == 2:
        opts = [(asc, nf), (not asc, not nf)]
    on = [(f"k{k}l", f"k{k}r") for k in range(nkeys)]
    _, out = run(split_batches(lrb, 700), split_batches(rrb, 500), on, jt, opts, NOSTAGE)
    compare(out, lrb, rrb, nkeys, jt, opts)


def presorted(rb, nkeys, opts):
    cols = V.from_batches([rb])
    perm = V.sort_permutation(cols, [(k, not a, nf) for k, (a, nf) in enumerate(opts[:nkeys])])
    out = rb.take(pa.array(perm))
    return out.set_column(nkeys, out.schema.names[nkeys], pa.array(np.arange(rb.num_rows, dtype=np.int64)))   # row ids of the sorted order


@pytest.mark.parametrize("jt", ALL_JT, ids=lambda j: JT_NAME[j])
@pytest.mark.parametrize("opts", [[(True, True)], [(False, False)]], ids=["asc", "desc"])
def test_streaming_left_batches_and_a_right_op_with_several_batches(jt, opts):
    """pre-sorted sides without a SortExec: the left in 37-row batches (key runs straddle them), the right op emits a batch per push"""
    rng = np.random.default_rng(7 + jt)
    lrb, rrb = presorted(side(rng, 4_000, "l", "i64", 1, 300, 0.05), 1, opts), presorted(side(rng, 2_500, "r", "i64", 1, 300, 0.05), 1, opts)
    _, out = run(split_batches(lrb, 37), split_batches(rrb, 211), [("k0l", "k0r")], jt, opts, NOSTAGE, sort_left=False, sort_right=False)
    compare(out, lrb, rrb, 1, jt, opts)


@pytest.mark.parametrize("jt", [PL.JOIN_RIGHT, PL.JOIN_FULL], ids=lambda j: JT_NAME[j])
def test_right_only_rows_settled_across_batches(jt):
    """right keys that no left key has, between and around left batches of one row each"""
    l = pa.RecordBatch.from_arrays([pa.array([2, 4, 4, 4, 9], pa.int64()), pa.array(np.arange(5, dtype=np.int64))], names=["k", "id"])
    r = pa.RecordBatch.from_arrays([pa.array([None, 1, 2, 3, 4, 5, 8, 9, 10, 11], pa.int64()), pa.array(np.arange(10, dtype=np.int64))], names=["rk", "rid"])
    _, out = run(split_batches(l, 1), [r], [("k", "rk")], jt, [(True, True)], NOSTAGE, sort_left=False, sort_right=False)
    rows = [tuple(x.values()) for b in out for x in b.to_pylist()]
    exp = [(None, None, None, 0), (None, None, 1, 1), (2, 0, 2, 2), (None, None, 3, 3), (4, 1, 4, 4), (4, 2, 4, 4), (4, 3, 4, 4),
           (None, None, 5, 5), (None, None, 8, 6), (9, 4, 9, 7), (None, None, 10, 8), (None, None, 11, 9)]
    assert rows == exp


def test_output_chunks_split_one_key_group():
    """one 300 x 300 key group (90 000 rows) emitted in chunks of at most 1 000 rows"""
    k_l = np.concatenate([np.arange(0, 50), np.full(300, 60), np.arange(70, 120)]).astype(np.int64)
    k_r = np.concatenate([np.arange(25, 55), np.full(300, 60), np.arange(100, 130)]).astype(np.int64)
    lrb = pa.RecordBatch.from_arrays([pa.array(k_l), pa.array(np.arange(len(k_l), dtype=np.int64))], names=["k0l", "idl"])
    rrb = pa.RecordBatch.from_arrays([pa.array(k_r), pa.array(np.arange(len(k_r), dtype=np.int64))], names=["k0r", "idr"])
    for jt in ALL_JT:
        _, out = run([lrb], [rrb], [("k0l", "k0r")], jt, [(True, True)], native.default_conf(staging_rows=0, max_launch_rows=1000))
        assert max(b.num_rows for b in out) <= 1000
        if jt == PL.JOIN_INNER:
            assert sum(b.num_rows for b in out) == 90_000 + 25 + 20
        compare(out, lrb, rrb, 1, jt, [(True, True)])


@pytest.mark.parametrize("jt", ALL_JT, ids=lambda j: JT_NAME[j])
def test_empty_sides_and_all_null_keys(jt):
    rng = np.random.default_rng(3)
    lrb, rrb = side(rng, 500, "l", "i32", 1, 20, 0.0), side(rng, 300, "r", "i32", 1, 20, 0.0)
    nulls = lambda rb: pa.RecordBatch.from_arrays([pa.nulls(rb.num_rows, rb.column(0).type)] + rb.columns[1:], names=rb.schema.names)
    for lb, rb in ((lrb, rrb.slice(0, 0)), (lrb.slice(0, 0), rrb), (lrb.slice(0, 0), rrb.slice(0, 0)), (nulls(lrb), rrb), (lrb, nulls(rrb)), (nulls(lrb), nulls(rrb))):
        _, out = run([lb], [rb], [("k0l", "k0r")], jt, [(True, False)], NOSTAGE, lschema=lrb.schema, rschema=rrb.schema)
        compare(out, lb, rb, 1, jt, [(True, False)])


# ---- unsorted input --------------------------------------------------------------------------------------------------------
def _ops(lrb, rrb, jt=PL.JOIN_INNER, opts=((True, True),), sort_right=False):
    plan = _plan([lrb], [rrb], [("k0l", "k0r")], jt, list(opts), sort_left=False, sort_right=sort_right)
    return plan, native.NativeOp(plan.plan_bytes(), NOSTAGE), native.NativeOp(plan.right.plan_bytes(), NOSTAGE)


def test_unsorted_left_is_refused():
    rng = np.random.default_rng(11)
    lrb, rrb = side(rng, 1_000, "l", "i64", 1, 50, 0.05), presorted(side(rng, 500, "r", "i64", 1, 50, 0.05), 1, [(True, True)])
    plan, op, rop = _ops(lrb, rrb)
    rop.push(rrb); rop.finish(); op.attach_right(rop)
    with pytest.raises(native.NativeError) as ei:
        op.push(lrb)
    assert ei.value.code == native.ERR_INVALID_ARG and "not sorted by the join keys" in ei.value.msg
    op.close(); rop.close()


def test_unsorted_across_a_batch_boundary_is_refused():
    l = pa.RecordBatch.from_arrays([pa.array([1, 2, 5], pa.int64()), pa.array([0, 1, 2], pa.int64())], names=["k0l", "idl"])
    l2 = pa.RecordBatch.from_arrays([pa.array([4, 6], pa.int64()), pa.array([3, 4], pa.int64())], names=["k0l", "idl"])
    r = pa.RecordBatch.from_arrays([pa.array([1, 5], pa.int64()), pa.array([0, 1], pa.int64())], names=["k0r", "idr"])
    plan, op, rop = _ops(l, r)
    rop.push(r); rop.finish(); op.attach_right(rop)
    op.push(l)
    with pytest.raises(native.NativeError) as ei:
        op.push(l2)
    assert ei.value.code == native.ERR_INVALID_ARG
    op.close(); rop.close()


@pytest.mark.parametrize("opts", [[(True, True)], [(False, True)], [(True, False)]])
def test_unsorted_right_is_refused_at_attach(opts):
    r = pa.RecordBatch.from_arrays([pa.array([None, 1, 3, 2], pa.int64()), pa.array([0, 1, 2, 3], pa.int64())], names=["k0r", "idr"])
    l = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([0], pa.int64())], names=["k0l", "idl"])
    plan, op, rop = _ops(l, r, opts=opts)
    rop.push(r); rop.finish()
    with pytest.raises(native.NativeError) as ei:
        op.attach_right(rop)
    assert ei.value.code == native.ERR_INVALID_ARG and "right input not sorted" in ei.value.msg
    op.close(); rop.close()


# ---- ABI misuse --------------------------------------------------------------------------------------------------------------
def _small():
    l = pa.RecordBatch.from_arrays([pa.array([1, 2, 2, 7], pa.int64()), pa.array([0, 1, 2, 3], pa.int64())], names=["k0l", "idl"])
    r = pa.RecordBatch.from_arrays([pa.array([2, 3, 7], pa.int64()), pa.array([0, 1, 2], pa.int64())], names=["k0r", "idr"])
    return l, r


def _code(fn):
    with pytest.raises(native.NativeError) as ei:
        fn()
    return ei.value.code


def test_push_or_finish_before_attach():
    l, r = _small()
    plan, op, rop = _ops(l, r)
    assert _code(lambda: op.push(l)) == native.ERR_STATE
    assert _code(op.finish) == native.ERR_STATE
    rop.push(r); rop.finish(); op.attach_right(rop)
    op.push(l); op.finish()
    assert sum(b.num_rows for b in op.pull_all()) == 3
    op.close(); rop.close()


def test_attach_misuse():
    l, r = _small()
    plan, op, rop = _ops(l, r)
    rop.push(r)
    assert _code(lambda: op.attach_right(rop)) == native.ERR_STATE                    # unfinished
    rop.finish()
    op.attach_right(rop)
    assert _code(lambda: op.attach_right(rop)) == native.ERR_STATE                    # twice
    assert _code(rop.pull) == native.ERR_STATE                                         # taken
    assert _code(rop.pull_device) == native.ERR_STATE
    rop.close()                                                                          # the batches outlive the right op
    op.push(l); op.finish()
    got = op.pull_all()
    assert [x["k0l"] for b in got for x in b.to_pylist()] == [2, 2, 7]
    op.close()


def test_attach_after_pull_and_other_ops():
    l, r = _small()
    plan, op, rop = _ops(l, r)
    rop.push(r); rop.finish()
    assert rop.pull() is not None
    assert _code(lambda: op.attach_right(rop)) == native.ERR_STATE                    # already pulled
    other = native.NativeOp(PL.MemoryExec.from_arrow([r]).plan_bytes(), NOSTAGE)
    other.push(r); other.finish()
    assert _code(lambda: rop.attach_right(other)) == native.ERR_STATE                 # not a join op
    bad_schema = pa.RecordBatch.from_arrays([pa.array([1], pa.int32()), pa.array([0], pa.int64())], names=["k0r", "idr"])
    wrong = native.NativeOp(PL.MemoryExec.from_arrow([bad_schema]).plan_bytes(), NOSTAGE)
    wrong.push(bad_schema); wrong.finish()
    assert _code(lambda: op.attach_right(wrong)) == native.ERR_INVALID_ARG
    for h in (op, rop, other, wrong):
        h.close()


# ---- fusion: SortExec -> SMJ -> Project -> AggExec(Partial) -> AggExec(Final) as one op ----------------------------------------------
@pytest.mark.parametrize("jt", [PL.JOIN_INNER, PL.JOIN_LEFT], ids=lambda j: JT_NAME[j])
def test_fused_sort_smj_project_agg(jt):
    rng = np.random.default_rng(21)
    lrb, rrb = side(rng, 20_000, "l", "i64", 1, 2_000, 0.02), side(rng, 8_000, "r", "i64", 1, 2_000, 0.02)
    smj = _plan(split_batches(lrb, 3_000), [rrb], [("k0l", "k0r")], jt, [(True, True)])
    proj = PL.ProjectExec([(E.Column("k0l"), "k"), (E.BinaryExpr(E.Column("vl"), "Plus", E.Column("vr")), "x")], smj)
    ins = proj.schema()
    g = [E.GroupingExpr("k", E.Column("k"))]
    aggs = lambda mode, ch: [E.AggExpr("s", mode, PL.create_agg(E.AGG_SUM, ch, ins, T.int64)), E.AggExpr("c", mode, PL.create_agg(E.AGG_COUNT, ch, ins, T.int64))]
    partial = PL.AggExec(PL.HashAgg, g, aggs(E.PARTIAL, [E.Column("x")]), False, proj)
    final = PL.AggExec(PL.HashAgg, g, aggs(E.FINAL, [E.placeholder(T.int64)]), False, partial)
    out = PL.collect(final, NOSTAGE)
    exp = V.join(V.from_batches([lrb]), V.from_batches([rrb]), [(0, 0)], jt, V.RIGHT_SIDE)
    k, v, w = exp[0], exp[2], exp[lrb.num_columns + 2]
    x_valid = v.valid & w.valid
    x = np.where(x_valid, v.values + w.values, 0)
    want = {}
    for kv, kk, xv, xx in zip(k.valid, k.values, x_valid, x):
        key = int(kk) if kv else None
        sm, c = want.get(key, (None, 0))
        if xv:
            sm = (sm or 0) + int(xx); c += 1
        want[key] = (sm, c)
    got = {r["k"]: (r["s"], r["c"]) for b in out for r in b.to_pylist()}
    assert got == want
    assert final.last_metrics["gpu_kernel_launches"] > 0
