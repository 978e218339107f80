"""Vectorized references of the hash join and the sort, for inputs of 10^6 to 10^8 rows.

numpy only, and no code shared with oracle/ (whose row-at-a-time restatements are too slow at these sizes;
tests/test_vector_ref.py checks the two against each other on small inputs).  A column is a VCol: raw values plus a
validity mask, bit-exact — f32 / f64 are kept as their IEEE bits, decimal128 as (low u64, high u64) pairs — and the
value of a NULL slot is set to 0, so two columns compare with np.array_equal.

Join: key equality on the integer values (int8 ... int64, date32, timestamp, and mixed widths all compare by value); a NULL
in any key never matches.  The pairs come from a stable argsort of the build keys, searchsorted and repeat.  Join types and
map sides use the wire numbering of blaze_b200.plans (JOIN_INNER ... JOIN_EXISTENCE, LEFT_SIDE / RIGHT_SIDE).

Sort: one order word per key column as unsigned 64-bit (integers: value XOR the sign bit; floats: IEEE totalOrder bits;
decimal128: the signed high word, then the low word; descending: bitwise NOT), a NULL rank before the words, and
np.lexsort for the stable permutation.
"""
from dataclasses import dataclass

import numpy as np
import pyarrow as pa

INNER, LEFT, RIGHT, FULL, SEMI, ANTI, EXISTENCE = range(7)            # blaze_b200.plans.JOIN_*
LEFT_SIDE, RIGHT_SIDE = 0, 1
SIGN64 = np.uint64(1 << 63)


@dataclass
class VCol:
    kind: str                  # "int" | "f32" | "f64" | "dec" | "bool"
    values: np.ndarray         # int: signed ints; f32 / f64: uint32 / uint64 bits; dec: (n, 2) uint64 (low, high); bool: uint8
    valid: np.ndarray          # bool

    def __len__(self):
        return len(self.valid)

    def take(self, idx):
        """idx < 0 gives a NULL row"""
        idx = np.asarray(idx, np.int64)
        none = idx < 0
        j = np.where(none, 0, idx)
        if len(self.valid) == 0:
            return VCol(self.kind, np.zeros((len(idx),) + self.values.shape[1:], self.values.dtype), np.zeros(len(idx), bool))
        return _zero_nulls(VCol(self.kind, self.values[j], self.valid[j] & ~none))


def _zero_nulls(c):
    if not c.valid.all():
        c.values = c.values.copy()
        c.values[~c.valid] = 0
    return c


def _kind_of(t):
    if pa.types.is_boolean(t):
        return "bool", None
    if pa.types.is_float32(t):
        return "f32", np.uint32
    if pa.types.is_float64(t):
        return "f64", np.uint64
    if pa.types.is_decimal(t):
        return "dec", np.uint64
    if pa.types.is_date32(t):
        return "int", np.int32
    if pa.types.is_timestamp(t):
        return "int", np.int64
    if pa.types.is_integer(t):
        return "int", t.to_pandas_dtype()
    raise TypeError(f"no VCol for {t}")


def col_from_arrow(arr) -> VCol:
    if isinstance(arr, pa.ChunkedArray):
        arr = pa.concat_arrays(arr.chunks) if arr.num_chunks else pa.array([], arr.type)
    n = len(arr)
    valid = np.ones(n, bool) if arr.null_count == 0 else np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), bool)
    kind, dt = _kind_of(arr.type)
    if kind == "bool":
        values = np.asarray(arr.fill_null(False).to_numpy(zero_copy_only=False), np.uint8)
    else:
        per = 2 if kind == "dec" else 1
        raw = np.frombuffer(arr.buffers()[1], dt, count=(arr.offset + n) * per)[arr.offset * per:]
        values = raw.reshape(n, 2).copy() if kind == "dec" else raw.copy()
    return _zero_nulls(VCol(kind, values, valid))


def from_batches(batches, ncols=None):
    """the columns of a list of pyarrow RecordBatches, concatenated; [] with ncols gives ncols empty columns"""
    if not batches:
        return [VCol("int", np.zeros(0, np.int64), np.zeros(0, bool)) for _ in range(ncols or 0)]
    return [col_from_arrow(pa.concat_arrays([b.column(i) for b in batches])) for i in range(batches[0].num_columns)]


def to_arrow(pa_type, values, valid=None):
    """an Arrow array from raw values (the bits are kept: NaN payloads, -0.0) and an optional validity mask"""
    values = np.ascontiguousarray(values)
    n = len(values)
    vbuf = None
    if valid is not None and not np.all(valid):
        vbuf = pa.py_buffer(np.packbits(np.asarray(valid, np.uint8), bitorder="little").tobytes())
    return pa.Array.from_buffers(pa_type, n, [vbuf, pa.py_buffer(values.tobytes())])


# ---- join ----------------------------------------------------------------------------------------------------------

def _key_ids(pkeys, bkeys):
    """one int64 per row whose equality is the equality of the key tuple; -> probe ids, probe valid, build ids, build valid"""
    pv = np.logical_and.reduce([c.valid for c in pkeys])
    bv = np.logical_and.reduce([c.valid for c in bkeys])
    if len(pkeys) == 1:
        return pkeys[0].values.astype(np.int64), pv, bkeys[0].values.astype(np.int64), bv
    both = np.concatenate([np.stack([c.values.astype(np.int64) for c in pkeys], 1), np.stack([c.values.astype(np.int64) for c in bkeys], 1)])
    _, inv = np.unique(both, axis=0, return_inverse=True)
    inv = inv.reshape(-1).astype(np.int64)
    np_ = len(pv)
    return inv[:np_], pv, inv[np_:], bv


def join(left, right, on, join_type, map_side):
    """left / right: lists of VCol; on: [(left column, right column)]; -> the output columns (left ++ right, or left
    [++ exists#0]) in some row order: compare with same_rows()"""
    build_is_left = map_side == LEFT_SIDE
    build, probe = (left, right) if build_is_left else (right, left)
    bk = [build[l if build_is_left else r] for l, r in on]
    pk = [probe[r if build_is_left else l] for l, r in on]
    pid, pv, bid, bv = _key_ids(pk, bk)
    nb, np_ = len(build[0]), len(probe[0])
    rows = np.nonzero(bv)[0]
    order = rows[np.argsort(bid[rows], kind="stable")]
    sorted_ids = bid[order]
    lo = np.searchsorted(sorted_ids, pid, "left")
    cnt = np.searchsorted(sorted_ids, pid, "right") - lo
    cnt[~pv] = 0
    probe_is_left = not build_is_left
    jt = join_type
    if jt in (SEMI, ANTI, EXISTENCE):
        if probe_is_left:                                             # the probe side is the join side
            matched, side, cols = cnt > 0, probe, probe
        else:
            matched = np.zeros(nb, bool)
            matched[order[np.repeat(lo, cnt) + _ranks(cnt)]] = True
            side, cols = build, build
        if jt == EXISTENCE:
            return list(cols) + [VCol("bool", matched.astype(np.uint8), np.ones(len(matched), bool))]
        keep = np.nonzero(matched if jt == SEMI else ~matched)[0]
        return [c.take(keep) for c in side]
    probe_outer = jt == FULL or (jt == LEFT and probe_is_left) or (jt == RIGHT and not probe_is_left)
    build_outer = jt == FULL or (jt == LEFT and not probe_is_left) or (jt == RIGHT and probe_is_left)
    pidx = np.repeat(np.arange(np_, dtype=np.int64), cnt)
    bidx = order[np.repeat(lo, cnt) + _ranks(cnt)].astype(np.int64)
    if probe_outer:
        un = np.nonzero(cnt == 0)[0]
        pidx, bidx = np.concatenate([pidx, un]), np.concatenate([bidx, np.full(len(un), -1, np.int64)])
    if build_outer:
        hit = np.zeros(nb, bool)
        hit[bidx[bidx >= 0]] = True
        un = np.nonzero(~hit)[0]
        pidx, bidx = np.concatenate([pidx, np.full(len(un), -1, np.int64)]), np.concatenate([bidx, un])
    pcols, bcols = [c.take(pidx) for c in probe], [c.take(bidx) for c in build]
    return bcols + pcols if build_is_left else pcols + bcols


def _ranks(cnt):
    """0, 1, ..., cnt[i] - 1 for every i, concatenated"""
    total = int(cnt.sum())
    starts = np.repeat(np.cumsum(cnt) - cnt, cnt)
    return np.arange(total, dtype=np.int64) - starts


# ---- sort ----------------------------------------------------------------------------------------------------------

def order_words(c: VCol, descending: bool):
    """the key's order words, most significant first, as uint64"""
    if c.kind == "int" or c.kind == "bool":
        words = [c.values.astype(np.int64).view(np.uint64) ^ SIGN64]
    elif c.kind == "f32":
        b = c.values.astype(np.uint64)
        words = [np.where(b >> np.uint64(31), ~b & np.uint64(0xFFFFFFFF), b | np.uint64(1 << 31))]
    elif c.kind == "f64":
        b = c.values
        words = [np.where(b >> np.uint64(63), ~b, b | SIGN64)]
    else:
        words = [c.values[:, 1] ^ SIGN64, c.values[:, 0].copy()]
    if descending:
        words = [~w for w in words]
    for w in words:
        w[~c.valid] = 0
    return words


def sort_permutation(cols, exprs):
    """exprs = [(column, descending, nulls_first)]; -> the stable permutation (np.int64)"""
    keys = []                                                           # most significant first
    for ci, desc, nulls_first in exprs:
        c = cols[ci]
        keys.append(np.where(c.valid, 1, 0 if nulls_first else 2).astype(np.uint8))
        keys += order_words(c, desc)
    if not keys or len(cols[0]) == 0:
        return np.arange(len(cols[0]) if cols else 0, dtype=np.int64)
    return np.lexsort(keys[::-1]).astype(np.int64)


def sort(cols, exprs, fetch=None):
    perm = sort_permutation(cols, exprs)
    if fetch is not None:
        perm = perm[:fetch]
    return [c.take(perm) for c in cols]


# ---- comparison ----------------------------------------------------------------------------------------------------

def canonical_order(cols, by=None):
    """a permutation that sorts the rows by the listed columns (default: all), validity and bits as keys"""
    keys = []
    for c in (cols if by is None else [cols[i] for i in by]):
        keys.append(c.valid.astype(np.uint8))
        keys += [c.values[:, 1], c.values[:, 0]] if c.kind == "dec" else [c.values.astype(np.int64) if c.kind != "bool" else c.values]
    n = len(cols[0]) if cols else 0
    if not keys or n == 0:
        return np.arange(n, dtype=np.int64)
    return np.lexsort(keys[::-1])


def assert_same_columns(got, exp, what=""):
    """row for row: the same values, validity and bits"""
    assert len(got) == len(exp), f"{what}{len(got)} columns, expected {len(exp)}"
    for i, (g, e) in enumerate(zip(got, exp)):
        assert len(g) == len(e), f"{what}column {i}: {len(g)} rows, expected {len(e)}"
        if len(e) == 0:
            continue
        bad = g.valid != e.valid
        if bad.any():
            r = int(np.nonzero(bad)[0][0])
            raise AssertionError(f"{what}column {i}: validity differs at {int(bad.sum())} rows, first row {r}: {g.valid[r]} vs {e.valid[r]}")
        gv, ev = g.values, e.values
        if gv.dtype != ev.dtype:
            gv, ev = gv.astype(np.int64), ev.astype(np.int64)
        bad = (gv != ev).reshape(len(e), -1).any(axis=1)
        if bad.any():
            r = int(np.nonzero(bad)[0][0])
            raise AssertionError(f"{what}column {i}: values differ at {int(bad.sum())} rows, first row {r}: {gv[r]} vs {ev[r]}")


def assert_same_rows(got, exp, by=None, what=""):
    """the same multiset of rows; `by` = columns that already make every row unique (e.g. row ids), or all columns"""
    if len(got) and len(exp) and len(got[0]) != len(exp[0]):
        raise AssertionError(f"{what}{len(got[0])} rows, expected {len(exp[0])}")
    pg, pe = canonical_order(got, by), canonical_order(exp, by)
    assert_same_columns([c.take(pg) for c in got], [c.take(pe) for c in exp], what)
