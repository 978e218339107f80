"""CPU restatement of the reference's ShuffleWriterExec path (SURVEY.md §8(f) rank 1) — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module; the product
(blaze_b200/) never does.  Every function cites the reference file:line it follows (paths relative to
the reference's native-engine/).

  radix_sort_by_key                datafusion-ext-commons/src/algorithm/rdx_sort.rs:23-73   (unstable American-flag sort)
  evaluate_*_partition_ids         datafusion-ext-plans/src/shuffle/mod.rs:163-275
  sort_batches_by_partition_id     datafusion-ext-plans/src/shuffle/buffered_data.rs:284-351
  BufferedData                     datafusion-ext-plans/src/shuffle/buffered_data.rs:48-282
  write_batch / read_batch         datafusion-ext-commons/src/io/batch_serde.rs:66-99,225-306,574-660
  IpcCompressionWriter / Reader    datafusion-ext-plans/src/common/ipc_compression.rs:34-183
  shuffle_write (no spills)        datafusion-ext-plans/src/shuffle/sort_repartitioner.rs:151-185

Pinned by the reference's own goldens (tests/test_shuffle_oracle.py): test_round_robin, test_range_partition,
test_range_partition_2 (buffered_data.rs:394-540, which also pin the unstable sort's row order), the rdx_sort fuzz
property (rdx_sort.rs:81-114) and the batch_serde / ipc_compression round trips (batch_serde.rs:662-713,
ipc_compression.rs:325-351).  The byte layout of batch_serde has no byte-level golden in the reference; it is pinned
by those round trips only.

Third-party pieces: the LZ4 *frame* codec is lz4_flex 0.11 in the reference (Cargo.toml); here pyarrow's "lz4" codec
(also the LZ4 frame format) plays that role — any conforming frame is readable by both.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from blaze_b200 import types as T
from blaze_b200.types import DataType, Schema
from oracle import blaze_oracle as O
from oracle.blaze_oracle import Batch, Col

BATCH_SIZE = 10000                       # datafusion-ext-commons/src/lib.rs:74-77
SUGGESTED_BATCH_MEM_SIZE = 8388608       # lib.rs:79-82
TARGET_BUF_SIZE = 4194304                # ipc_compression.rs:77-80 (SHUFFLE_COMPRESSION_TARGET_BUF_SIZE default)


# =====================================================================================================================
# rdx_sort.rs:23-73
# =====================================================================================================================
def radix_sort_by_key(array: list, num_keys: int, key: Callable) -> List[int]:
    """In-place; returns counts.  The element order inside a bucket is whatever the swap sequence leaves (unstable)."""
    counts = [0] * num_keys
    for item in array:
        counts[key(item)] += 1
    cur = [0] * num_keys
    end = [0] * num_keys
    beg = 0
    for idx, c in enumerate(counts):
        if c > 0:
            cur[idx], end[idx] = beg, beg + c
            beg += c
    inexhausted = list(range(num_keys))
    while True:
        inexhausted = [i for i in inexhausted if cur[i] < end[i]]
        if len(inexhausted) <= 1:
            break
        for part_idx in inexhausted:
            c, e = cur[part_idx], end[part_idx]          # captured before the inner loop, as the reference does
            for item_idx in range(c, e):
                t = key(array[item_idx])
                array[item_idx], array[cur[t]] = array[cur[t]], array[item_idx]
                cur[t] += 1
    return counts


# =====================================================================================================================
# shuffle/mod.rs: Partitioning + partition ids
# =====================================================================================================================
@dataclass
class SortKey:
    col: int
    descending: bool = False
    nulls_first: bool = True             # arrow SortOptions::default()


@dataclass
class Partitioning:
    kind: str                            # "hash" | "round_robin" | "single" | "range"
    n: int = 1
    hash_cols: Sequence[int] = ()        # column indices (the reference evaluates PhysicalExprs; columns on this path)
    sort_keys: Sequence[SortKey] = ()
    bounds: Sequence[tuple] = ()         # range: n-1 bound rows, each a tuple of python values (None = NULL)

    def partition_count(self) -> int:    # mod.rs:124-132
        return 1 if self.kind == "single" else self.n


def _row_cmp(a: tuple, b: tuple, keys: Sequence[SortKey]) -> int:
    """byte order of arrow-row encoded rows == lexicographic order under each field's SortOptions"""
    for x, y, k in zip(a, b, keys):
        if x is None or y is None:
            if x is None and y is None:
                continue
            less = (x is None) == k.nulls_first
            return -1 if less else 1
        if x != y:
            lt = x < y
            if k.descending:
                lt = not lt
            return -1 if lt else 1
    return 0


def _binary_search(bounds, target, keys) -> int:        # mod.rs:258-275
    low, high = 0, len(bounds) - 1
    while low <= high:
        mid = (low + high) >> 1
        c = _row_cmp(bounds[mid], target, keys)
        if c < 0:
            low = mid + 1
        elif c > 0:
            high = mid - 1
        else:
            return mid
    return low


def get_partition(key_row: tuple, bounds, keys) -> int:  # mod.rs:234-256 (ascending = true at the only call site)
    n = len(bounds)
    if n <= 128:
        p = 0
        while p < n and _row_cmp(key_row, bounds[p], keys) > 0:
            p += 1
    else:
        p = min(_binary_search(bounds, key_row, keys), n)
    return p


def _cell(c: Col, r: int):
    if not c.valid[r]:
        return None
    v = c.values[r]
    return v.item() if hasattr(v, "item") else v


def evaluate_partition_ids(p: Partitioning, batch: Batch, round_robin_start: int = 0) -> np.ndarray:
    n = batch.num_rows
    if p.kind == "hash":                                 # mod.rs:163-188
        hashes = O.create_murmur3_hashes([batch.cols[i] for i in p.hash_cols], n, 42)
        return O.partition_ids(hashes, p.n)
    if p.kind == "round_robin":                          # mod.rs:190-202
        return ((np.arange(n, dtype=np.int64) + round_robin_start) % p.n).astype(np.uint32)
    if p.kind == "range":                                # mod.rs:204-232
        keys = list(p.sort_keys)
        return np.array([get_partition(tuple(_cell(batch.cols[k.col], r) for k in keys), p.bounds, keys) for r in range(n)], np.uint32)
    if p.kind == "single":
        return np.zeros(n, np.uint32)
    raise ValueError(p.kind)


# =====================================================================================================================
# buffered_data.rs:284-351
# =====================================================================================================================
def interleave(batches: Sequence[Batch], indices: Sequence[Tuple[int, int]]) -> Batch:
    schema = batches[0].schema
    cols = []
    for ci in range(len(schema)):
        dt = schema[ci].dtype
        vals = O._zeros(dt, len(indices))
        valid = np.zeros(len(indices), bool)
        for o, (b, r) in enumerate(indices):
            vals[o] = batches[b].cols[ci].values[r]
            valid[o] = batches[b].cols[ci].valid[r]
        cols.append(Col(dt, vals, valid))
    return Batch(schema, cols, len(indices))


def sort_batches_by_partition_id(batches: Sequence[Batch], p: Partitioning, current_num_rows: int, partition_id: int):
    """-> (partition_offsets[n+1], sorted_batch)"""
    num_partitions = p.partition_count()
    rr = (partition_id * 1000193 + current_num_rows) % num_partitions
    triples = []
    for bi, b in enumerate(batches):
        pids = evaluate_partition_ids(p, b, rr)
        if p.kind == "round_robin":
            rr = (rr + b.num_rows) % num_partitions
        triples.extend((int(pid), bi, ri) for ri, pid in enumerate(pids))
    counts = radix_sort_by_key(triples, num_partitions, lambda t: t[0])
    offsets = [0]
    for c in counts:
        offsets.append(offsets[-1] + c)
    if not batches:
        return offsets, None
    return offsets, interleave(batches, [(b, r) for _, b, r in triples])


# =====================================================================================================================
# io/mod.rs:60-83 + io/batch_serde.rs
# =====================================================================================================================
write_len = O.write_len
read_len = O.read_len

_WIDTH = {T.INT8: 1, T.INT16: 2, T.INT32: 4, T.INT64: 8, T.FLOAT32: 4, T.FLOAT64: 8, T.DATE32: 4, T.TIMESTAMP_US: 8, T.DECIMAL128: 16}
_NPDT = {T.INT8: "<i1", T.INT16: "<i2", T.INT32: "<i4", T.INT64: "<i8", T.FLOAT32: "<f4", T.FLOAT64: "<f8", T.DATE32: "<i4", T.TIMESTAMP_US: "<i8"}


def _values_le_bytes(c: Col) -> np.ndarray:
    """(n, width) uint8 matrix of the little-endian values (NULL slots as stored: 0)"""
    n = len(c)
    w = _WIDTH[c.dtype.id]
    if c.dtype.id == T.DECIMAL128:
        raw = b"".join((int(v) if ok else 0).to_bytes(16, "little", signed=True) for v, ok in zip(c.values, c.valid))
        return np.frombuffer(raw, np.uint8).reshape(n, 16)
    vals = np.where(c.valid, c.values, 0).astype(_NPDT[c.dtype.id])
    return np.frombuffer(vals.tobytes(), np.uint8).reshape(n, w)


def _write_nulls(c: Col, has_nulls: Optional[bool]) -> bytes:
    """batch_serde.rs:274-284: `1` + repacked validity bits when the array carries a null buffer, else `0`.  Whether an
    all-valid array carries one is a property of how it was built (not a wire contract): has_nulls=None means
    "iff some row is NULL"."""
    n = len(c)
    present = (not bool(c.valid.all())) if has_nulls is None else has_nulls
    if not present:
        return write_len(0)
    return write_len(1) + np.packbits(np.asarray(c.valid, np.uint8), bitorder="little").tobytes()[: (n + 7) // 8]


def write_array(c: Col, has_nulls: Optional[bool] = None) -> bytes:
    n = len(c)
    dt = c.dtype.id
    if dt == T.NULLTYPE:                                             # batch_serde.rs:115
        return b""
    out = _write_nulls(c, has_nulls)
    if dt == T.BOOL:                                                 # :530-551 bits, never transposed
        return out + np.packbits(np.asarray(c.values, bool).astype(np.uint8), bitorder="little").tobytes()[: (n + 7) // 8]
    if dt == T.BINARY:                                               # :574-600 + write_offsets :225-248
        lens = np.array([len(v) if ok else 0 for v, ok in zip(c.values, c.valid)], "<i4")
        lens_t = np.frombuffer(lens.tobytes(), np.uint8).reshape(n, 4).T.tobytes() if n else b""
        return out + lens_t + b"".join(bytes(v) for v, ok in zip(c.values, c.valid) if ok)
    m = _values_le_bytes(c)                                          # :264-306: byte planes when width > 1
    return out + (m.T.tobytes() if m.shape[1] > 1 else m.tobytes())


def write_batch(num_rows: int, cols: Sequence[Col], has_nulls: Optional[Sequence[Optional[bool]]] = None) -> bytes:
    """batch_serde.rs:66-77"""
    out = write_len(num_rows)
    for i, c in enumerate(cols):
        assert len(c) == num_rows
        out += write_array(c, None if has_nulls is None else has_nulls[i])
    return out


def _read_nulls(buf: bytes, pos: int, n: int):
    has, pos = read_len(buf, pos)
    if has != 1:
        return np.ones(n, bool), pos
    nb = (n + 7) // 8
    bits = np.unpackbits(np.frombuffer(buf, np.uint8, nb, pos), bitorder="little")[:n].astype(bool)
    return bits, pos + nb


def read_array(buf: bytes, pos: int, dt: DataType, n: int) -> Tuple[Col, int]:
    if dt.id == T.NULLTYPE:
        return Col(dt, np.zeros(n, np.int8), np.zeros(n, bool)), pos
    valid, pos = _read_nulls(buf, pos, n)
    if dt.id == T.BOOL:
        nb = (n + 7) // 8
        vals = np.unpackbits(np.frombuffer(buf, np.uint8, nb, pos), bitorder="little")[:n].astype(bool)
        return Col(dt, vals, valid), pos + nb
    if dt.id == T.BINARY:
        lens = np.frombuffer(np.frombuffer(buf, np.uint8, 4 * n, pos).reshape(4, n).T.tobytes(), "<i4") if n else np.zeros(0, "<i4")
        pos += 4 * n
        vals = np.empty(n, object)
        for i in range(n):
            vals[i] = bytes(buf[pos: pos + int(lens[i])]); pos += int(lens[i])
        return Col(dt, vals, valid), pos
    w = _WIDTH[dt.id]
    raw = np.frombuffer(buf, np.uint8, w * n, pos)
    rows = (raw.reshape(w, n).T if w > 1 else raw.reshape(n, 1)).tobytes()
    pos += w * n
    if dt.id == T.DECIMAL128:
        vals = np.empty(n, object)
        for i in range(n):
            vals[i] = int.from_bytes(rows[16 * i: 16 * i + 16], "little", signed=True)
    else:
        vals = np.frombuffer(rows, _NPDT[dt.id]).astype(O._NP[dt.id]).copy()
    return Col(dt, vals, valid), pos


def read_batch(buf: bytes, pos: int, schema: Schema) -> Tuple[Optional[Batch], int]:
    """batch_serde.rs:79-99; (None, pos) at end of input"""
    if pos >= len(buf):
        return None, pos
    n, pos = read_len(buf, pos)
    cols = []
    for f in schema:
        c, pos = read_array(buf, pos, f.dtype, n)
        cols.append(c)
    return Batch(schema, cols, n), pos


# =====================================================================================================================
# common/ipc_compression.rs
# =====================================================================================================================
def _lz4_frame_compress(data: bytes) -> bytes:
    import pyarrow as pa
    return pa.Codec("lz4").compress(data, asbytes=True)


def _lz4_frame_decompress(data: bytes) -> bytes:
    import pyarrow as pa
    return pa.CompressedInputStream(pa.BufferReader(data), "lz4").read()


class IpcCompressionWriter:
    """ipc_compression.rs:34-112: blocks of `u32 LE length ‖ LZ4 frame`, a block is closed when its compressed buffer
    reaches 0.9 x 4 MiB (checked after each batch) or on finish_current_buf()."""

    def __init__(self, compress: Callable[[bytes], bytes] = _lz4_frame_compress):
        self.out = bytearray()
        self._pending = bytearray()
        self._compress = compress

    def write_batch(self, num_rows: int, cols: Sequence[Col]):
        if num_rows == 0:
            return
        self._pending += write_batch(num_rows, cols)
        # the reference looks at the *compressed* length so far; a streaming encoder's internal buffering makes the exact
        # cut point codec-specific and unobservable to a reader: cut on the compressed size of what is pending
        if len(self._compress(bytes(self._pending))) + 4 >= TARGET_BUF_SIZE * 0.9:
            self.finish_current_buf()

    def finish_current_buf(self):
        if self._pending:
            frame = self._compress(bytes(self._pending))
            self.out += struct.pack("<I", len(frame)) + frame
            self._pending = bytearray()

    def count(self) -> int:
        return len(self.out)


def read_ipc_blocks(data: bytes) -> bytes:
    """IpcCompressionReader (ipc_compression.rs:114-183): the concatenated decompressed block payloads"""
    pos, out = 0, bytearray()
    while pos < len(data):
        (blen,) = struct.unpack_from("<I", data, pos); pos += 4
        out += _lz4_frame_decompress(bytes(data[pos: pos + blen])); pos += blen
    return bytes(out)


def read_partition(data: bytes, schema: Schema) -> List[Batch]:
    """what the reduce side's IpcReaderExec does with one partition's byte range"""
    raw = read_ipc_blocks(data)
    pos, out = 0, []
    while True:
        b, pos = read_batch(raw, pos, schema)
        if b is None:
            return out
        out.append(b)


# =====================================================================================================================
# BufferedData (buffered_data.rs:48-282) + SortShuffleRepartitioner::shuffle_write without spills
# =====================================================================================================================
def batch_mem_size(b: Batch) -> int:
    """get_batch_mem_size (datafusion-ext-commons/src/arrow/array_size.rs): buffer bytes; only steers batching"""
    total = 0
    for c in b.cols:
        if c.dtype.id == T.BINARY:
            total += 4 * (b.num_rows + 1) + sum(len(v) for v in c.values)
        elif c.dtype.id == T.BOOL:
            total += (b.num_rows + 7) // 8
        else:
            total += _WIDTH.get(c.dtype.id, 0) * b.num_rows
        total += (b.num_rows + 7) // 8
    return total


def compute_suggested_batch_size_for_output(mem_size: int, num_rows: int) -> int:      # lib.rs:93-116
    if num_rows == 0:
        return BATCH_SIZE
    est = max(mem_size, 16) // max(num_rows, 1)
    return max(20, min(BATCH_SIZE, SUGGESTED_BATCH_MEM_SIZE // max(est, 16)))


@dataclass
class BufferedData:
    partitioning: Partitioning
    partition_id: int
    staging: List[Batch] = field(default_factory=list)
    staging_num_rows: int = 0
    staging_mem_used: int = 0
    sorted_batches: List[Batch] = field(default_factory=list)
    sorted_offsets: List[List[int]] = field(default_factory=list)
    num_rows: int = 0
    sorted_mem_used: int = 0

    def add_batch(self, b: Batch):                                                      # :88-101
        self.num_rows += b.num_rows
        self.staging_num_rows += b.num_rows
        self.staging_mem_used += batch_mem_size(b) * 2
        self.staging.append(b)
        if self.staging_mem_used > compute_suggested_batch_size_for_output(self.staging_mem_used, self.staging_num_rows):
            self.flush_staging()

    def flush_staging(self):                                                            # :103-119
        sorted_num_rows = self.num_rows - self.staging_num_rows
        offsets, sb = sort_batches_by_partition_id(self.staging, self.partitioning, sorted_num_rows, self.partition_id)
        self.staging, self.staging_num_rows, self.staging_mem_used = [], 0, 0
        self.sorted_mem_used += batch_mem_size(sb) + len(offsets) * 4
        self.sorted_batches.append(sb)
        self.sorted_offsets.append(offsets)

    def write(self) -> Tuple[bytes, List[int]]:                                         # :123-158 -> (data, offsets[n+1])
        n = self.partitioning.partition_count()
        if self.num_rows == 0:
            return b"", [0] * (n + 1)
        if self.staging:
            self.flush_staging()
        sub = compute_suggested_batch_size_for_output(self.sorted_mem_used + self.staging_mem_used, self.num_rows)
        w = IpcCompressionWriter()
        offsets: List[int] = []
        for pid in range(n):                                                            # OffsettedMergeIterator: partition by partition,
            idx = [(bi, r) for bi, offs in enumerate(self.sorted_offsets) for r in range(offs[pid], offs[pid + 1])]   # run by run
            if not idx:
                continue
            offsets += [w.count()] * (pid + 1 - len(offsets))
            for s in range(0, len(idx), sub):
                chunk = interleave(self.sorted_batches, idx[s: s + sub])
                w.write_batch(chunk.num_rows, chunk.cols)
            w.finish_current_buf()
        offsets += [w.count()] * (n + 1 - len(offsets))
        return bytes(w.out), offsets


def shuffle_write(batches: Sequence[Batch], p: Partitioning, partition_id: int = 0) -> Tuple[bytes, bytes]:
    """sort_repartitioner.rs:151-185 (no spills): -> (.data bytes, .index bytes = (n+1) little-endian i64 offsets)"""
    bd = BufferedData(p, partition_id)
    for b in batches:
        bd.add_batch(b)
    data, offsets = bd.write()
    return data, b"".join(struct.pack("<q", o) for o in offsets)


def read_shuffle_file(data: bytes, index: bytes, schema: Schema) -> List[List[Batch]]:
    offs = struct.unpack("<%dq" % (len(index) // 8), index)
    return [read_partition(data[offs[i]: offs[i + 1]], schema) for i in range(len(offs) - 1)]
