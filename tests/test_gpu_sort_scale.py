"""SortExec at scale and at the edges of every key type, against the vectorized reference (tests/vector_ref.py).  The radix
passes are stable (kernels_sort.cu), so every case compares the WHOLE output row for row with the stable reference: values,
validity and float bits.  Covers several tiles per CTA (5 x 10^6 rows), sizes around the 4096-row tile, 10^3 pushed batches
with and without validity, NaNs of both signs and with payloads, ±0, subnormals, decimal words beyond 64 bits, digits that
never vary (constant, all-NULL, one differing row, i << 40), six keys at once and fetch around the tile size."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import exprs as E, native, plans as PL
import vector_ref as V

pytestmark = pytest.mark.gpu

TYPES = {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "date32": pa.date32(), "ts": pa.timestamp("us"),
         "f32": pa.float32(), "f64": pa.float64(), "dec": pa.decimal128(38, 0)}
F64_EDGES = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF00000DEADBEEF, 0x7FF4000000000123, 0x7FF0000000000000,
                      0xFFF0000000000000, 0, 1 << 63, 1, (1 << 63) | 1, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF], np.uint64)
F32_EDGES = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF812345, 0x7FA00042, 0x7F800000, 0xFF800000, 0, 1 << 31, 1, (1 << 31) | 1,
                      0x7F7FFFFF, 0xFF7FFFFF], np.uint32)
DEC_EDGES = [10**38 - 1, -(10**38 - 1), 2**64, -(2**64), 2**64 + 1, 2**100, -(2**100), 2**63 - 1, 2**63, -(2**63), -(2**63) - 1, -1, 0, 1]


def _np_type(t):
    return np.int32 if pa.types.is_date32(t) else np.int64 if pa.types.is_timestamp(t) else t.to_pandas_dtype()


def _dec_raw(vals):
    vals = [int(v) for v in vals]
    return np.array([[v & (2**64 - 1), (v >> 64) & (2**64 - 1)] for v in vals], np.uint64).reshape(-1, 2)


def _edge_values(rng, t, n):
    """random values, half of them replaced by the type's edge values"""
    pick = rng.random(n) < 0.5
    if pa.types.is_decimal(t):
        v = rng.integers(-2**62, 2**62, (n, 2)).view(np.uint64)
        v[:, 1] = np.where(rng.random(n) < 0.5, 0, np.uint64(2**64 - 1))                # mostly inside the 64-bit range ...
        e = _dec_raw(DEC_EDGES)                                                            # ... and the edges outside it
        v[pick] = e[rng.integers(0, len(e), int(pick.sum()))]
        return v
    if pa.types.is_float32(t):
        v = rng.normal(size=n).astype(np.float32).view(np.uint32)
        v[pick] = F32_EDGES[rng.integers(0, len(F32_EDGES), int(pick.sum()))]
        return v
    if pa.types.is_float64(t):
        v = rng.normal(size=n).view(np.uint64)
        v[pick] = F64_EDGES[rng.integers(0, len(F64_EDGES), int(pick.sum()))]
        return v
    dt = _np_type(t)
    info = np.iinfo(dt)
    v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
    e = np.array([info.min, info.max, -1, 0, 1, info.min + 1, info.max - 1], dt)
    v[pick] = e[rng.integers(0, len(e), int(pick.sum()))]
    return v


def _col(rng, t, n, null_frac):
    return V.to_arrow(t, _edge_values(rng, t, n), rng.random(n) >= null_frac if null_frac else None)


def _run(batches, exprs, fetch=None):
    names = batches[0].schema.names
    plan = PL.SortExec(PL.MemoryExec.from_arrow(batches, batches[0].schema), [(E.Column(names[c]), d, nf) for c, d, nf in exprs], fetch)
    return PL.collect(plan, native.default_conf(staging_rows=0))


def _check(batches, exprs, fetch=None):
    out = _run(batches, exprs, fetch)
    exp = V.sort(V.from_batches(batches), exprs, fetch)
    V.assert_same_columns(V.from_batches(out, batches[0].num_columns), exp)
    return exp


def _rows(n):
    return V.to_arrow(pa.int64(), np.arange(n, dtype=np.int64))


# ---- every key type, both directions, NULLs first and last ---------------------------------------------------------

@pytest.mark.parametrize("nulls", ["nulls_first", "nulls_last"])
@pytest.mark.parametrize("order", ["asc", "desc"])
@pytest.mark.parametrize("key", list(TYPES))
def test_key_types_at_their_edges(key, order, nulls):
    rng = np.random.default_rng(list(TYPES).index(key))
    n = 30_000
    rb = pa.RecordBatch.from_arrays([_col(rng, TYPES[key], n, 0.1), _rows(n), _col(rng, pa.float64(), n, 0.1)], names=["k", "row", "x"])
    _check([rb.slice(0, 9_999), rb.slice(9_999)], [(0, order == "desc", nulls == "nulls_first")])


def test_decimal_words():
    """±(10^38 - 1), |x| >= 2^64, 2^63 - 1 against 2^63 (they differ only in the top bit of the low word) and -1 against 0"""
    vals = np.array(DEC_EDGES * 50, object)
    np.random.default_rng(1).shuffle(vals)
    n = len(vals)
    rb = pa.RecordBatch.from_arrays([V.to_arrow(pa.decimal128(38, 0), _dec_raw(vals)), _rows(n)], names=["d", "row"])
    for desc in (False, True):
        _check([rb], [(0, desc, True)])
    got = V.sort(V.from_batches([rb]), [(0, False, True)])[0].values
    as_int = [int(lo) | (int(hi) << 64) for lo, hi in got]
    as_int = [v - 2**128 if v >= 2**127 else v for v in as_int]
    assert as_int == sorted(as_int)                                          # the reference's order is the numeric order


# ---- sizes ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [5_000_000, 4096 * 7 - 1, 4096 * 7 + 1, 4096 * 64 + 1, 255, 1])
def test_sizes(n):
    """5 x 10^6 rows: several 4096-row tiles per CTA; sizes one off the tile; fewer than 256 rows"""
    rng = np.random.default_rng(n % 1000)
    rb = pa.RecordBatch.from_arrays([_col(rng, pa.int32(), n, 0.05), _col(rng, pa.float64(), n, 0.05), _rows(n)], names=["a", "b", "row"])
    step = max(1, n // 3 + 1)
    _check([rb.slice(i, step) for i in range(0, n, step)], [(0, True, False), (1, False, True)])


def test_a_thousand_batches_with_and_without_validity():
    """10^3 pushed batches of 5 000 rows; some carry NULLs in the key, the others no validity buffer at all"""
    rng = np.random.default_rng(1000)
    batches = []
    for b in range(1_000):
        n = 5_000
        k = V.to_arrow(pa.int64(), rng.integers(-2**40, 2**40, n), (rng.random(n) > 0.2) if b % 3 == 0 else None)
        batches.append(pa.RecordBatch.from_arrays([k, V.to_arrow(pa.int64(), np.arange(b * n, (b + 1) * n, dtype=np.int64))], names=["k", "row"]))
    _check(batches, [(0, False, False)])


# ---- digits that never vary ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", ["constant", "all_null", "one_differs", "shift40", "one_null"])
@pytest.mark.parametrize("key", ["i64", "f64", "dec", "i16"])
def test_digits_that_never_vary(key, shape):
    """a constant key runs no pass and keeps the input order; an all-NULL key; one row that differs; int64 i << 40 whose low
    five bytes never vary; exactly one NULL (its NULL-rank pass must run)"""
    rng = np.random.default_rng(len(shape))
    n, t = 20_000, TYPES[key]
    raw = _edge_values(rng, t, 1).repeat(n, axis=0).reshape((n, 2) if key == "dec" else n)
    valid = np.ones(n, bool)
    if shape == "all_null":
        valid[:] = False
    elif shape == "one_differs":
        raw[12_345] = _edge_values(np.random.default_rng(99), t, 1)[0] if key != "i16" else raw[0] ^ 1
    elif shape == "shift40":
        raw = (rng.integers(-2**23, 2**23, n).astype(np.int64) << 40).astype(_np_type(t)) if key in ("i64", "i16") else raw
    elif shape == "one_null":
        valid[777] = False
    rb = pa.RecordBatch.from_arrays([V.to_arrow(t, raw, valid if not valid.all() else None), _rows(n)], names=["k", "row"])
    for desc, nf in ((False, True), (True, False)):
        exp = _check([rb.slice(0, 7_001), rb.slice(7_001)], [(0, desc, nf)])
        if shape == "constant":
            assert (exp[1].values == np.arange(n)).all()


# ---- many keys and every payload width -----------------------------------------------------------------------------

def test_six_keys_and_payloads_of_every_width():
    rng = np.random.default_rng(6)
    n = 200_000
    small = lambda t, k: V.to_arrow(t, rng.integers(0, k, n).astype(_np_type(t)), rng.random(n) > 0.1)
    keys = [small(pa.int8(), 3), small(pa.int16(), 4), _col(rng, pa.float32(), n, 0.1), small(pa.date32(), 5), _col(rng, pa.decimal128(38, 0), n, 0.1),
            small(pa.int64(), 2)]
    payload = [_col(rng, t, n, 0.2) for t in (pa.int8(), pa.int16(), pa.int32(), pa.float64(), pa.decimal128(38, 0))]
    rb = pa.RecordBatch.from_arrays(keys + payload + [_rows(n)], names=[f"c{i}" for i in range(12)])
    exprs = [(0, False, True), (1, True, False), (2, False, False), (3, True, True), (4, False, True), (5, True, False)]
    _check([rb.slice(0, 65_537), rb.slice(65_537)], exprs)


@pytest.mark.parametrize("fetch", ["0", "1", "4095", "4097", "n-1", "n", "n+1"])
def test_fetch(fetch):
    rng = np.random.default_rng(7)
    n = 12_289
    f = eval(fetch)
    rb = pa.RecordBatch.from_arrays([_col(rng, pa.int64(), n, 0.1), _col(rng, pa.float32(), n, 0.1), _rows(n)], names=["a", "b", "row"])
    batches = [rb.slice(0, 4_000), rb.slice(4_000, 5_003), rb.slice(9_003)]
    if f == 0:
        assert _run(batches, [(0, True, False)], 0) == []
        return
    _check(batches, [(0, True, False), (1, False, True)], f)
