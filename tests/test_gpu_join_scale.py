"""The hash join at production shapes against the vectorized reference (tests/vector_ref.py): unique build keys (the fused
probe + gather path of PK-FK joins) at 10^3 and 3 x 10^6 probe rows, payloads of every width with NULLs pushed at odd
offsets, sides of 16 / 17 / 33 columns, keys at their integer extremes and of mixed widths, probe clusters that wrap
around the table, one key duplicated 10^6 times, a probe batch above the 2^26-row split, and output counts beyond
2^31 - 1 rows, which are refused."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL
import vector_ref as V

pytestmark = pytest.mark.gpu

JT = {"inner": PL.JOIN_INNER, "left": PL.JOIN_LEFT, "right": PL.JOIN_RIGHT, "full": PL.JOIN_FULL, "semi": PL.JOIN_SEMI, "anti": PL.JOIN_ANTI,
      "existence": PL.JOIN_EXISTENCE}
SIDE = {"mapL": PL.LEFT_SIDE, "mapR": PL.RIGHT_SIDE}
PAYLOAD = [pa.int8(), pa.int16(), pa.int32(), pa.date32(), pa.float32(), pa.int64(), pa.float64(), pa.timestamp("us"), pa.decimal128(38, 0)]


def _np_type(t):
    return np.int32 if pa.types.is_date32(t) else np.int64 if pa.types.is_timestamp(t) else t.to_pandas_dtype()


def _payload(rng, t, n, null_frac=0.1):
    valid = rng.random(n) >= null_frac
    if pa.types.is_decimal(t):
        return V.to_arrow(t, rng.integers(-2**63, 2**63 - 1, (n, 2), dtype=np.int64).view(np.uint64), valid)
    if pa.types.is_floating(t):
        return V.to_arrow(t, rng.normal(size=n).astype(_np_type(t)), valid)
    info = np.iinfo(_np_type(t))
    return V.to_arrow(t, rng.integers(info.min, info.max, n, dtype=_np_type(t), endpoint=True), valid)


def _table(rng, tag, keys, key_valid=None, payload=(), key_type=pa.int32(), lead=0):
    """columns k<tag>, id<tag> (the row's position), then the payload; `lead` extra rows in front that are sliced off again"""
    n = len(keys) + lead
    keys = np.concatenate([np.zeros(lead, np.int64), np.asarray(keys, np.int64)]).astype(_np_type(key_type))
    kv = None if key_valid is None else np.concatenate([np.ones(lead, bool), key_valid])
    cols = [V.to_arrow(key_type, keys, kv), V.to_arrow(pa.int64(), np.arange(n, dtype=np.int64) - lead)] + [_payload(rng, t, n) for t in payload]
    return pa.RecordBatch.from_arrays(cols, names=[f"k{tag}", f"id{tag}"] + [f"p{tag}{i}" for i in range(len(payload))])


def _slices(rb, first, step):
    """rb[first:] as batches of `step` rows: with odd `first` and `step` the batches start at every bit offset of a byte"""
    return [rb.slice(i, min(step, rb.num_rows - i)) for i in range(first, rb.num_rows, step)]


def _run(lb, rb, on, jt, map_side):
    left, right = PL.MemoryExec.from_arrow(lb, lb[0].schema), PL.MemoryExec.from_arrow(rb, rb[0].schema)
    schema = PL.build_join_schema(left.schema(), right.schema(), jt)
    plan = PL.BroadcastJoinExec(schema, left, right, [(E.Column(l), E.Column(r)) for l, r in on], jt, map_side)
    return PL.collect(plan, native.default_conf(staging_rows=0)), len(schema)      # staging_rows=0: batches are imported as they are, offsets included


def _check(lb, rb, on, jt, map_side):
    """the GPU's rows == the reference's rows; the id columns make every output row unique, so they alone order the rows"""
    nl, names_l, names_r = lb[0].num_columns, lb[0].schema.names, rb[0].schema.names
    on_idx = [(names_l.index(a), names_r.index(b)) for a, b in on]
    out, ncols = _run(lb, rb, on, jt, map_side)
    exp = V.join(V.from_batches(lb), V.from_batches(rb), on_idx, jt, map_side)
    by = [names_l.index("idl")] + ([] if jt in (PL.JOIN_SEMI, PL.JOIN_ANTI, PL.JOIN_EXISTENCE) else [nl + names_r.index("idr")])
    got = V.from_batches(out, ncols)
    V.assert_same_rows(got, exp, by)
    return got


def _sides(map_side, build, probe):
    return (build, probe) if map_side == PL.LEFT_SIDE else (probe, build)


# ---- unique build keys: lookup pass + fused gather ----------------------------------------------------------------

@pytest.mark.parametrize("rows", ["n1e3", "n3e6"])
@pytest.mark.parametrize("match", ["m0", "m50", "m100"])
@pytest.mark.parametrize("side", list(SIDE))
@pytest.mark.parametrize("jt", ["inner", "left", "right", "full"])
def test_unique_build_keys(jt, side, match, rows):
    """payloads of every width with NULLs on both sides; probe and build NULL keys (NULL-key build rows are not in the
    map and come back unmatched under RIGHT / FULL); batches at odd offsets; 3 x 10^6 rows = several tiles per CTA"""
    rng = np.random.default_rng(["inner", "left", "right", "full"].index(jt) * 100 + len(side) * 10 + len(match) + len(rows))
    map_side = SIDE[side]
    bt, pt = ("l", "r") if map_side == PL.LEFT_SIDE else ("r", "l")
    n, nb = (1_000, 1_000) if rows == "n1e3" else (3_000_000, 250_000)
    bkeys = rng.permutation(nb).astype(np.int64) * 7 + 3
    bvalid = rng.random(nb) >= 0.02
    frac = {"m0": 0.0, "m50": 0.5, "m100": 1.0}[match]
    live = bkeys[bvalid]
    pkeys = np.where(rng.random(n) < frac, live[rng.integers(0, len(live), n)], rng.integers(0, nb, n) * 7 + 5)
    pvalid = np.ones(n, bool) if frac == 1.0 else rng.random(n) >= 0.02
    build = _slices(_table(rng, bt, bkeys, bvalid, PAYLOAD, lead=5), 5, 301 if nb == 1_000 else 77_777)
    probe = _slices(_table(rng, pt, pkeys, pvalid, PAYLOAD, lead=3), 3, 333 if n == 1_000 else 999_997)
    lb, rb = _sides(map_side, build, probe)
    got = _check(lb, rb, [("kl", "kr")], JT[jt], map_side)
    if frac == 1.0 and jt == "inner":
        assert len(got[0]) == n


@pytest.mark.parametrize("where", ["probe", "build"])
@pytest.mark.parametrize("ncols", [16, 17, 33])
def test_side_column_counts(ncols, where):
    """16 columns a side take the fused gather; 17 and 33 take the pair path, whose gathers run 16 columns at a time"""
    rng = np.random.default_rng(ncols)
    n, nb = 20_000, 5_000
    wide = [PAYLOAD[i % len(PAYLOAD)] for i in range(ncols - 2)]
    bkeys = rng.permutation(nb).astype(np.int64)
    build = _table(rng, "r", bkeys, rng.random(nb) > 0.05, wide if where == "build" else PAYLOAD[:2], lead=1)
    probe = _table(rng, "l", rng.integers(-100, nb + 100, n), rng.random(n) > 0.05, wide if where == "probe" else PAYLOAD[:2], lead=7)
    for jt in ("inner", "full"):
        _check(_slices(probe, 7, 4_999), _slices(build, 1, 2_047), [("kl", "kr")], JT[jt], PL.RIGHT_SIDE)


def test_unique_keys_but_one_pair():
    """10^6 unique build keys plus one duplicate in a second batch: the most duplicated key has 2 rows, so the probe takes the
    pair path and must return both partners"""
    rng = np.random.default_rng(3)
    nb = 1_000_000
    bkeys = np.concatenate([rng.permutation(nb), [123_457]]).astype(np.int64)
    build = _table(rng, "r", bkeys, payload=[pa.int16()])
    probe = _table(rng, "l", np.concatenate([rng.integers(0, 2 * nb, 200_000), [123_457]]), payload=[pa.float64()])
    got = _check([probe], [build.slice(0, 600_001), build.slice(600_001)], [("kl", "kr")], PL.JOIN_INNER, PL.RIGHT_SIDE)
    assert (got[0].values == 123_457).sum() >= 2


# ---- keys --------------------------------------------------------------------------------------------------------

KEY_TYPES = {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64()}


@pytest.mark.parametrize("side", list(SIDE))
@pytest.mark.parametrize("types", ["i8-i8", "i16-i16", "i32-i32", "i64-i64", "i32-i64", "i8-i64"])
def test_integer_keys_at_their_extremes(types, side):
    """MIN, MAX, -1 and 0 of every width; across widths the keys compare by value: int8 5 does not meet int64 261"""
    lt, rt = (KEY_TYPES[t] for t in types.split("-"))
    rng = np.random.default_rng(len(types) + len(side))
    li, ri = np.iinfo(lt.to_pandas_dtype()), np.iinfo(rt.to_pandas_dtype())
    edges = np.array([li.min, li.max, -1, 0, 1, li.min + 1, li.max - 1], np.int64)
    aliases = np.array([v for v in (ri.min, ri.max, 256 + 5, -256 - 1, 65536 + 7, 2**32 - 1, 2**32, li.max + 1, li.min - 1) if ri.min <= v <= ri.max], np.int64)
    lkeys = np.concatenate([edges, rng.integers(li.min, li.max, 3_000, endpoint=True), [5, 7, -1]])
    rkeys = np.unique(np.concatenate([edges, aliases, rng.integers(max(li.min, ri.min) // 2, min(li.max, ri.max) // 2, 500)]))
    left = _table(rng, "l", lkeys, rng.random(len(lkeys)) > 0.03, [pa.int32()], key_type=lt)
    right = _table(rng, "r", rng.permutation(rkeys), None, [pa.int64()], key_type=rt)
    for jt in ("inner", "full"):
        _check([left], [right], [("kl", "kr")], JT[jt], SIDE[side])


def test_two_keys_in_both_orders():
    """(a, b) and (b, a) are different keys"""
    rng = np.random.default_rng(4)
    a, b = rng.integers(-2**40, 2**40, 5_000), rng.integers(-3, 3, 5_000)
    def t(tag, x, y):
        rb = _table(rng, tag, x, rng.random(len(x)) > 0.02, [pa.int16()], key_type=pa.int64())
        return pa.RecordBatch.from_arrays(list(rb.columns) + [V.to_arrow(pa.int64(), np.asarray(y, np.int64), rng.random(len(x)) > 0.02)], names=rb.schema.names + [f"j{tag}"])
    for side in SIDE.values():
        bt, pt = ("l", "r") if side == PL.LEFT_SIDE else ("r", "l")
        build = t(bt, np.concatenate([a, b[:100]]), np.concatenate([b, a[:100]]))
        probe = t(pt, np.concatenate([b, a, a]), np.concatenate([a, b, b]))
        lb, rb = _sides(side, [build], [probe])
        for jt in ("inner", "full", "semi", "existence"):
            _check(lb, rb, [("kl", "kr"), ("jl", "jr")], JT[jt], side)


def _slot(keys, mask):
    """restates key_hash of kernels_join.cu for one int64 key column (only to choose colliding keys)"""
    w = np.asarray(keys, np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        h = w * np.uint64(0x9E3779B97F4A7C15)
    return (((h >> np.uint64(32)) ^ (h >> np.uint64(13))) & np.uint64(0xFFFFFFFF) & np.uint64(mask)).astype(np.int64)


def test_probe_clusters_that_wrap_around_the_table():
    """400 build keys share a home slot 4 slots before the end of the table, so inserting and probing them walks a long
    cluster that wraps past slot 0; 400 absent keys with the same home slot walk the whole cluster before they miss.
    The keys are chosen with a restatement of key_hash: if the hash changes the test stays correct but loses its bite."""
    nb = 3_000
    cap = 1024
    while cap < 2 * nb:
        cap <<= 1
    target = cap - 4
    cand = np.arange(1, 20_000_000, dtype=np.int64)
    same = cand[_slot(cand, cap - 1) == target]
    assert len(same) >= 800
    cluster, absent = same[:400], same[400:800]
    rng = np.random.default_rng(5)
    others = np.setdiff1d(rng.choice(np.arange(-10**7, 0, dtype=np.int64), nb - 400, replace=False), cluster)
    build = _table(rng, "r", rng.permutation(np.concatenate([cluster, others])), payload=[pa.int64()], key_type=pa.int64())
    probe = _table(rng, "l", rng.permutation(np.concatenate([cluster, absent, others[:1000], cluster])), payload=[pa.int32()], key_type=pa.int64())
    for jt in ("inner", "left", "anti"):
        _check([probe], [build], [("kl", "kr")], JT[jt], PL.RIGHT_SIDE)


@pytest.mark.parametrize("hot_rows", [1, 3])
@pytest.mark.parametrize("jt", ["inner", "full"])
def test_one_key_a_million_times(jt, hot_rows):
    rng = np.random.default_rng(hot_rows)
    hot = -7
    bkeys = rng.permutation(np.concatenate([np.arange(100_000), np.full(1_000_000, hot)])).astype(np.int64)
    build = _table(rng, "r", bkeys, payload=[pa.int16()])
    pkeys = rng.permutation(np.concatenate([np.full(hot_rows, hot), rng.integers(-1_000, 110_000, 20_000)]))
    probe = _table(rng, "l", pkeys, (rng.random(len(pkeys)) > 0.01) | (pkeys == hot),[pa.float32()])
    got = _check([probe], _slices(build, 0, 333_333), [("kl", "kr")], JT[jt], PL.RIGHT_SIDE)
    assert (got[0].values[got[0].valid] == hot).sum() == hot_rows * 1_000_000


# ---- the 2^26-row split of a probe batch --------------------------------------------------------------------------

@pytest.fixture(scope="module")
def huge_probe():
    rng = np.random.default_rng(26)
    n = (1 << 26) + 12_345
    keys = rng.integers(0, 2_000, n + 3)
    t = _table(rng, "l", keys[3:], rng.random(n) > 0.05, [pa.int16()], lead=3)
    build = _table(rng, "r", rng.permutation(1_000).astype(np.int64) * 2, payload=[pa.int8()])
    return t.slice(3, n), build


@pytest.mark.parametrize("jt", ["inner", "left", "semi", "anti", "existence"])
def test_probe_batch_above_the_2_26_split(huge_probe, jt):
    """one batch of 2^26 + 12 345 rows at bit offset 3: its second chunk reaches every probe kernel (and the Existence copy)
    with a column offset above 2^26 that is not a multiple of 8"""
    probe, build = huge_probe
    _check([probe], [build], [("kl", "kr")], JT[jt], PL.RIGHT_SIDE)


# ---- output counts ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hot_build():
    rng = np.random.default_rng(21)
    return _table(rng, "r", np.full(1 << 21, 42, np.int64))


@pytest.mark.parametrize("probe_rows", [2048, 1100])
def test_more_than_2_31_output_rows_are_refused(hot_build, probe_rows):
    """2^21 build rows of one key probed by 2048 rows of that key = 2^32 output rows: one tile's count must not wrap to 0
    (which returned no rows); 1100 rows = 2.3 x 10^9 output rows"""
    probe = _table(np.random.default_rng(1), "l", np.full(probe_rows, 42, np.int64))
    with pytest.raises(native.NativeError) as ei:
        _run([probe], [hot_build], [("kl", "kr")], PL.JOIN_INNER, PL.RIGHT_SIDE)
    assert ei.value.code == native.ERR_UNSUPPORTED


def test_one_probe_row_of_a_2_21_row_key(hot_build):
    probe = _table(np.random.default_rng(1), "l", np.full(1, 42, np.int64))
    got = _check([probe], [hot_build], [("kl", "kr")], PL.JOIN_INNER, PL.RIGHT_SIDE)
    assert len(got[0]) == 1 << 21
