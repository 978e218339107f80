"""ParquetScanExec at the edges of its decode and of its row-group pruning.

The oracle is pyarrow's libparquet reading the same file (tests/helpers.py: assert_same_table compares types, validity and the
bits of every non-NULL slot).  Decimals are also checked against the unscaled integers of the written decimal.Decimal values, so
that a writer and a reader agreeing on a wrong value cannot pass.  Every test asserts, from the file's metadata or from its page
headers (read by the small Thrift walker below, independent of parquet_meta.cc), that the file has the encoding or page layout the
test is about: a change of writer defaults must fail here, not quietly turn a case into a no-op.

  decimals         every precision 1..38 as INT32 / INT64 / FIXED_LEN_BYTE_ARRAY of 1..16 bytes, at the magnitude limits and leading bytes
  fixed width      int8..int64, date32 and timestamp[us] at their limits; float / double zeros, infinities, subnormals, NaN payloads
  index widths     dictionaries of 1 (bit width 0) .. 2^20+ entries, widths growing page by page, fallback to PLAIN mid-chunk
  run tables       one page per stored value (a run per lane), NULL runs of 1..1000, row groups of 1..4097 rows, v1 / v2, Booleans PLAIN / RLE
  refusals         encodings, types and codecs outside the GPU path raise ERR_UNSUPPORTED; the next scan still decodes
  pruning          a few hundred seeded predicates: the rows match pyarrow's filter, and the row groups kept match a count from the statistics
"""
import decimal
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from blaze_b200 import exprs as E, native, plans as PL, types as T
from helpers import assert_same_table, parquet_scan, value_slots

pytestmark = pytest.mark.gpu

PLAIN, RLE, RLE_DICTIONARY = 0, 3, 8           # parquet Encoding enum values in page headers
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DEC_CTX = decimal.Context(prec=60)                 # exact scaling of 38-digit values (the default context rounds to 28 digits)


# ---- page headers ---------------------------------------------------------------------------------------------------------
class _Thrift:
    """The part of Thrift's compact protocol a PageHeader needs: integers, booleans and nested structs; binaries, doubles and
    containers are skipped."""

    def __init__(self, b, p):
        self.b, self.p = b, p

    def byte(self):
        self.p += 1
        return self.b[self.p - 1]

    def varint(self):
        v = s = 0
        while True:
            x = self.byte()
            v |= (x & 0x7F) << s
            s += 7
            if not x & 0x80:
                return v

    def zigzag(self):
        v = self.varint()
        return (v >> 1) ^ -(v & 1)

    def value(self, t):
        if t in (1, 2):                                   # a Boolean field: the value is in the type nibble
            return t == 1
        if t == 3:
            return self.byte()
        if t in (4, 5, 6):
            return self.zigzag()
        if t == 7:
            self.p += 8
        elif t == 8:
            n = self.varint()
            self.p += n
        elif t in (9, 10):
            h = self.byte()
            n = h >> 4 if h >> 4 != 15 else self.varint()
            for _ in range(n):
                self.byte() if h & 0x0F in (1, 2) else self.value(h & 0x0F)
        elif t == 11:
            n = self.varint()
            kv = self.byte() if n else 0
            for _ in range(n):
                self.value(kv >> 4), self.value(kv & 0x0F)
        elif t == 12:
            return self.struct()
        else:
            raise AssertionError(f"thrift type {t}")

    def struct(self):
        out, fid = {}, 0
        while True:
            h = self.byte()
            if h == 0:
                return out
            fid = fid + (h >> 4) if h >> 4 else self.zigzag()
            out[fid] = self.value(h & 0x0F)


def _pages(path, rg=0, col=0):
    """The pages of one column chunk: [{kind, num_values, encoding, num_nulls (v2), bit_width (dictionary-encoded pages of an
    uncompressed chunk), at (file offset of the body)}]."""
    md = pq.ParquetFile(path).metadata
    cc = md.row_group(rg).column(col)
    optional = md.schema.column(col).max_definition_level > 0
    start = cc.dictionary_page_offset if cc.has_dictionary_page else cc.data_page_offset
    with open(path, "rb") as f:
        f.seek(start)
        data = f.read(cc.total_compressed_size)
    out, p = [], 0
    while p < len(data):
        r = _Thrift(data, p)
        h = r.struct()
        body, p = r.p, r.p + h[3]
        kind = {0: "v1", 2: "dict", 3: "v2"}[h[1]]
        sub = h[{"v1": 5, "dict": 7, "v2": 8}[kind]]
        pg = {"kind": kind, "num_values": sub[1], "encoding": sub[4] if kind == "v2" else sub[2], "at": start + body}
        if kind == "v2":
            pg["num_nulls"] = sub[2]
        if kind != "dict" and optional and cc.compression == "UNCOMPRESSED":     # where the definition levels (RLE / bit-packed hybrid) lie
            pg["levels_at"], pg["levels_len"] = (start + body, sub.get(5, 0)) if kind == "v2" else (start + body + 4, int.from_bytes(data[body: body + 4], "little"))
        if kind != "dict" and pg["encoding"] == RLE_DICTIONARY and cc.compression == "UNCOMPRESSED":
            if kind == "v2":
                vo = sub.get(5, 0) + sub.get(6, 0)
            else:
                vo = 4 + int.from_bytes(data[body: body + 4], "little") if optional else 0
            if body + vo < p:                                   # an all-NULL page stores no bit width
                pg["bit_width"], pg["bit_width_at"] = data[body + vo], start + body + vo
        out.append(pg)
    return out


def _data_pages(path, rg=0, col=0):
    return [p for p in _pages(path, rg, col) if p["kind"] != "dict"]


def _scan_all(path, schema, **kw):
    plan = parquet_scan(path, schema, **kw)
    return PL.collect(plan), plan.last_metrics


def _check_file(path, schema=None):
    """scan the whole file and compare with libparquet; returns the scan's output as one table"""
    out, _ = _scan_all(path, schema or pq.read_schema(path))
    exp = pq.read_table(path)
    assert_same_table(out, exp)
    return pa.Table.from_batches(out, schema=out[0].schema) if out else exp.slice(0, 0)


def _chunks(path, name):
    md = pq.ParquetFile(path).metadata
    i = md.schema.names.index(name)
    return [md.row_group(g).column(i) for g in range(md.num_row_groups)]


# ---- 1. decimals at every storage width ----------------------------------------------------------------------------------
def _flba_width(p):
    """the bytes libparquet stores a decimal of precision p in: the fewest that hold +-(10^p - 1) in two's complement"""
    return next(w for w in range(1, 17) if 10 ** p - 1 < 1 << (8 * w - 1))


def _decimal_cases():
    for p in range(1, 39):
        for as_int in ((True, False) if p <= 18 else (False,)):
            yield pytest.param(p, as_int, id=f"p{p}-{'int' if as_int else 'flba'}")


def _decimal_unscaled(p, width):
    """0, +-1, +-(10^p - 1), +-10^(p-1), and the values of the stored width whose leading byte is 0x7F, 0x80, 0xFF or 0x00
    (both ends of each such range) where the precision holds them"""
    big = 10 ** p - 1
    vals = {0, 1, -1, big, -big, 10 ** (p - 1), -10 ** (p - 1)}
    step = 1 << (8 * (width - 1))
    for lead in (0x7F, 0x80, 0xFF, 0x00):
        for u in (lead * step, lead * step + step - 1, lead * step + step // 2 + 1):
            v = u - (1 << (8 * width)) if u >> (8 * width - 1) else u
            if abs(v) <= big:
                vals.add(v)
    return sorted(vals)


@pytest.mark.parametrize("p,as_int", list(_decimal_cases()))
def test_decimal_storage_widths(tmp_path, p, as_int):
    s = p // 3
    width = (4 if p <= 9 else 8) if as_int else _flba_width(p)
    unscaled = _decimal_unscaled(p, width)
    rng = np.random.default_rng(p)
    rows = [unscaled[i] for i in rng.permutation(np.tile(np.arange(len(unscaled)), 3))]
    null = np.arange(len(rows)) % 3 == 1
    ty = pa.decimal128(p, s)
    dec = lambda m: pa.array([None if m is not None and m[i] else decimal.Decimal(v).scaleb(-s, DEC_CTX) for i, v in enumerate(rows)], ty)
    t = pa.table({"plain": dec(None), "plain_null": dec(null), "dict": dec(None), "dict_null": dec(null)})
    path = str(tmp_path / "d.parquet")
    pq.write_table(t, path, use_dictionary=["dict", "dict_null"], store_decimal_as_integer=as_int, compression="none")

    f = pq.ParquetFile(path)
    physical = {4: "INT32", 8: "INT64"}[width] if as_int else "FIXED_LEN_BYTE_ARRAY"
    for i, name in enumerate(t.schema.names):
        col = f.schema.column(i)
        assert col.physical_type == physical and (as_int or col.length == width), col
        cc = f.metadata.row_group(0).column(i)
        assert cc.has_dictionary_page == name.startswith("dict") and ("RLE_DICTIONARY" in cc.encodings) == name.startswith("dict"), (name, cc)
    lead = {(v & ((1 << 8 * width) - 1)) >> (8 * width - 8) for v in unscaled}
    assert {0x00, 0xFF} <= lead, lead

    got = _check_file(path)
    for name, m in (("plain", None), ("plain_null", null), ("dict", None), ("dict_null", null)):
        slots = value_slots(got.column(name).combine_chunks())
        as_ints = [int.from_bytes(bytes(r), "little", signed=True) for r in slots]
        exp = [0 if m is not None and m[i] else v for i, v in enumerate(rows)]         # unscaled value of the written Decimal; zero under a NULL
        assert as_ints == exp, name


# ---- 2. fixed-width edges ------------------------------------------------------------------------------------------------
F64_BITS = [0x0, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000,          # +-0, +-inf
            0x1, 0x800FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF,   # subnormals, smallest / largest normal
            0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000001, 0x7FFFFFFFFFFFFFFF,    # quiet NaNs, both signs, payloads
            0x7FF0000000000001, 0xFFF4000000000ABC, 0x7FF4000000000000, 0x3FF0000000000000]   # signalling NaNs; 1.0
F32_BITS = [0x0, 0x80000000, 0x7F800000, 0xFF800000, 0x1, 0x807FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF,
            0x7FC00000, 0xFFC00000, 0x7FC00001, 0x7FFFFFFF, 0x7F800001, 0xFFA00ABC, 0x7FA00000, 0x3F800000]


def _int_edges(bits):
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    return [lo, lo + 1, -1, 0, hi - 1, hi]


def _edge_table(n_rep, rng):
    cols = {
        "i8": pa.array(_int_edges(8), pa.int8()), "i16": pa.array(_int_edges(16), pa.int16()),
        "i32": pa.array(_int_edges(32), pa.int32()), "i64": pa.array(_int_edges(64), pa.int64()),
        "d": pa.array(_int_edges(32), pa.int32()).cast(pa.date32()),                   # date32 over its whole int32 range
        "ts": pa.array(_int_edges(64), pa.int64()).cast(pa.timestamp("us")),
        "f32": pa.array(np.array(F32_BITS, np.uint32).view(np.float32)), "f64": pa.array(np.array(F64_BITS, np.uint64).view(np.float64)),
    }
    out = {}
    n = max(len(a) for a in cols.values()) * n_rep
    for name, a in cols.items():
        idx = rng.permutation(np.resize(np.arange(len(a)), n))               # every edge n_rep times or more, in a random order
        out[name] = a.take(pa.array(idx))
        out[name + "_n"] = pc.if_else(pa.array(np.arange(n) % 4 == 1), pa.scalar(None, a.type), out[name])
    return pa.table(out)


@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
@pytest.mark.parametrize("dictionary", [False, True], ids=["plain", "dict"])
def test_fixed_width_edges(tmp_path, dictionary, page_version):
    t = _edge_table(5, np.random.default_rng(7))
    path = str(tmp_path / "e.parquet")
    pq.write_table(t, path, use_dictionary=dictionary, data_page_version=page_version, data_page_size=1, write_batch_size=64, compression="none")
    for i, name in enumerate(t.schema.names):
        pages = _data_pages(path, 0, i)
        assert len(pages) > 1 and all(pg["kind"] == ("v1" if page_version == "1.0" else "v2") for pg in pages), name
        assert all(pg["encoding"] == (RLE_DICTIONARY if dictionary else PLAIN) for pg in pages), (name, [pg["encoding"] for pg in pages])
    got = _check_file(path)
    if not dictionary:                                # PLAIN stores the input bits: the scan returns them (NaN payloads and signs included)
        for name in t.schema.names:
            a, g = t.column(name).combine_chunks(), got.column(name).combine_chunks()
            v = a.is_valid().to_numpy(zero_copy_only=False)
            assert np.array_equal(value_slots(g)[v], value_slots(a)[v]), name


# ---- 3. dictionary index widths ------------------------------------------------------------------------------------------
DICT_SIZES = [1, 2, 3, 4, 5, 255, 256, 257, 65535, 65536, 65537, (1 << 20) + 3]


@pytest.mark.parametrize("k", DICT_SIZES, ids=[f"{k}entries" for k in DICT_SIZES])
def test_dictionary_index_widths(tmp_path, k):
    rng = np.random.default_rng(k)
    n = max(2 * k, 5000)
    entries = rng.choice(1 << 40, size=k, replace=False).astype(np.int64) - (1 << 39)
    idx = np.arange(n) % k                                          # every entry, the last one (all index bits set) included
    t = pa.table({"x": pa.array(entries[idx]), "x_n": pa.array(entries[idx], mask=(np.arange(n) % 7 == 3) & (np.arange(n) >= k))})   # NULLs after the first pass
    path = str(tmp_path / "k.parquet")
    pq.write_table(t, path, use_dictionary=True, dictionary_pagesize_limit=1 << 30, data_page_size=32 << 10, row_group_size=n, compression="none")
    final = (k - 1).bit_length()
    for c in range(2):
        pages = _pages(path, 0, c)
        assert pages[0]["kind"] == "dict" and pages[0]["num_values"] == k
        data = pages[1:]
        assert all(pg["encoding"] == RLE_DICTIONARY for pg in data), "a PLAIN data page: the dictionary fell back"
        assert max(pg["bit_width"] for pg in data) == max(final, 1), [pg["bit_width"] for pg in data]
    if k == 1:
        # libparquet writes bit width 1 for a one-entry dictionary.  Width 0 (every index is 0 and takes no bits) is valid Parquet:
        # rewrite the width byte of each page of the required column, whose indices are one RLE run of 0 stored in one byte
        # that a reader of width 0 must not consume
        blob = bytearray(open(path, "rb").read())
        for pg in _data_pages(path, 0, 0):
            assert blob[pg["bit_width_at"]] == 1 and blob[pg["bit_width_at"] + 1] & 1 == 0      # width 1, then an RLE run header
            blob[pg["bit_width_at"]] = 0
        open(path, "wb").write(bytes(blob))
        assert all(pg["bit_width"] == 0 for pg in _data_pages(path, 0, 0))
        assert pq.read_table(path).column("x").equals(t.column("x"))
    got = _check_file(path)
    assert got.column("x").equals(t.column("x"))


def test_dictionary_width_grows_across_pages_and_falls_back_mid_chunk(tmp_path):
    n = 60_000
    rng = np.random.default_rng(11)
    grow = rng.permutation(n // 2).astype(np.int64)[np.arange(n) // 2]                # a new entry every second row: wider indices page by page
    t = pa.table({"grow": pa.array(grow, mask=np.arange(n) % 5 == 0),
                  "fallback": pa.array(rng.integers(-2**62, 2**62, n), mask=np.arange(n) % 9 == 0)})    # unique: the dictionary page limit is hit
    path = str(tmp_path / "g.parquet")
    pq.write_table(t, path, use_dictionary=True, dictionary_pagesize_limit=320 << 10, data_page_size=4 << 10, row_group_size=n, compression="none")
    pages = _data_pages(path, 0, 0)
    widths = [pg["bit_width"] for pg in pages]
    assert all(pg["encoding"] == RLE_DICTIONARY for pg in pages) and widths == sorted(widths) and len(set(widths)) >= 4, widths
    enc = [pg["encoding"] for pg in _data_pages(path, 0, 1)]
    first_plain = enc.index(PLAIN)
    assert first_plain >= 2 and set(enc[:first_plain]) == {RLE_DICTIONARY} and set(enc[first_plain:]) == {PLAIN}, enc
    _check_file(path)


# ---- 4. run tables: one page per stored value, NULL runs, row-group sizes --------------------------------------------------
NULL_RUNS = [1, 7, 8, 9, 31, 32, 33, 1000]


def _null_mask(pattern, n):
    if pattern == "none":
        return np.zeros(n, bool)
    if pattern == "alternating":
        return np.arange(n) % 2 == 1
    m = []
    for i, run in enumerate(NULL_RUNS * (n // 1000 + 1)):          # a NULL run, then a valid run of a different length
        m += [True] * run + [False] * (1, 3, 8, 9, 2, 33, 5, 64)[i % 8]
    return np.array(m[:n])


def _poison_level_padding(path, col):
    """Set the unused bits of every partial last bit-packed group of definition levels to 1 in place.  The spec leaves those padding
    bits unspecified and a reader must stop at the page's value count; returns the number of pages changed."""
    blob, changed = bytearray(open(path, "rb").read()), 0
    for pg in _data_pages(path, 0, col):
        p, end, got = pg["levels_at"], pg["levels_at"] + pg["levels_len"], 0
        while got < pg["num_values"] and p < end:
            r = _Thrift(blob, p)
            h = r.varint()
            p = r.p
            if h & 1:                                          # bit-packed: (h >> 1) groups of 8 one-bit levels
                for i in range(pg["num_values"] - got, (h >> 1) * 8):
                    blob[p + i // 8] |= 1 << (i % 8)
                    changed += i == pg["num_values"] - got
                got += (h >> 1) * 8
                p += h >> 1
            else:
                got += h >> 1
                p += 1
    open(path, "wb").write(bytes(blob))
    return changed


def _all_null_pages_between_valid(path, col, mask):
    """row group 0 of the column has a page holding only NULLs with pages holding values before and after it"""
    pages = _data_pages(path, 0, col)
    rows = np.cumsum([0] + [pg["num_values"] for pg in pages])
    all_null = [mask[rows[i]: rows[i + 1]].all() for i in range(len(pages))]
    return any(all_null[i] and not all(all_null[:i]) and not all(all_null[i + 1:]) for i in range(len(pages)))


def _all_types_table(n, mask, rng):
    m = mask if mask.any() else None
    dec = lambda p, s, hi: pa.array([decimal.Decimal(int(v)).scaleb(-s) for v in rng.integers(-hi, hi, n)], pa.decimal128(p, s), mask=m)
    return pa.table({
        "i8": pa.array(rng.integers(-128, 128, n).astype(np.int8), mask=m), "i16": pa.array(rng.integers(-2**15, 2**15, n).astype(np.int16), mask=m),
        "i32": pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32), mask=m), "i64": pa.array(rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64), mask=m),
        "f32": pa.array(rng.normal(size=n).astype(np.float32), mask=m), "f64": pa.array(rng.normal(size=n), mask=m),
        "d": pa.array(rng.integers(-20000, 20000, n).astype(np.int32), mask=m).cast(pa.date32()),
        "ts": pa.array(rng.integers(-2**60, 2**60, n, dtype=np.int64), mask=m).cast(pa.timestamp("us")),
        "dec9": dec(9, 2, 10**9 - 1), "dec18": dec(18, 3, 10**18 - 1), "dec30": dec(30, 4, 10**18),
        "i64_dict": pa.array(rng.integers(-5, 5, n, dtype=np.int64), mask=m), "dec30_dict": dec(30, 0, 3),
        "b_plain": pa.array(rng.random(n) < 0.5, mask=m), "b_rle": pa.array(rng.random(n) < 0.5, mask=m),
        "all_null": pa.array([None] * n, pa.int32()), "no_null": pa.array(rng.integers(-9, 9, n, dtype=np.int64)),
    })


@pytest.mark.parametrize("pattern", ["none", "alternating", "runs"])
@pytest.mark.parametrize("rg", [1, 7, 8, 9, 31, 32, 33, 4095, 4097])
@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
def test_one_page_per_row(tmp_path, page_version, rg, pattern):
    n = 8300 if rg > 1000 else 1300 if rg > 9 else 300               # rows: at least two row groups, at most ~300 of them
    mask = _null_mask(pattern, n)
    t = _all_types_table(n, mask, np.random.default_rng(rg))
    path = str(tmp_path / "r.parquet")
    dict_cols = ["i64_dict", "dec30_dict"]
    pq.write_table(t, path, data_page_size=1, write_batch_size=1, row_group_size=rg, data_page_version=page_version, compression="none",
                   use_dictionary=dict_cols, column_encoding={c: ("RLE" if c == "b_rle" else "PLAIN") for c in t.schema.names if c not in dict_cols})
    md = pq.ParquetFile(path).metadata
    assert md.num_row_groups == -(-n // rg)
    names = t.schema.names
    rows, stored = min(rg, n), int((~mask[:rg]).sum())
    for name in ("i32", "dec30", "b_plain"):                        # PLAIN: a page ends at every stored value
        pages = _data_pages(path, 0, names.index(name))
        assert sum(pg["num_values"] for pg in pages) == rows and len(pages) >= stored and {pg["encoding"] for pg in pages} == {PLAIN}, name
    for name, enc in (("b_rle", RLE), ("i64_dict", RLE_DICTIONARY), ("no_null", PLAIN)):    # RLE-encoded values: a page per row, NULL rows too
        pages = _data_pages(path, 0, names.index(name))
        assert len(pages) == rows and {pg["encoding"] for pg in pages} == {enc}, (name, len(pages))
    if (pattern == "alternating" and rg > 2) or (pattern == "runs" and rg > 30):                           # the first row group has valid rows after a NULL run
        assert _all_null_pages_between_valid(path, names.index("b_rle"), mask)
    assert all(c.statistics.null_count == c.num_values and not c.statistics.has_min_max for c in _chunks(path, "all_null"))   # no value runs at all
    assert md.schema.column(names.index("no_null")).max_definition_level == 1 and all(c.statistics.null_count == 0 for c in _chunks(path, "no_null"))
    _check_file(path)


@pytest.mark.parametrize("page_rows", [7, 13, 1000])
@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
def test_level_runs_and_partial_bit_packed_groups(tmp_path, page_version, page_rows):
    """pages and row groups of sizes that are not multiples of 8 (a partial last bit-packed group), long RLE level runs next to
    bit-packed ones, all-NULL pages between valid pages, Booleans crossing page boundaries"""
    n = 20_003
    mask = _null_mask("runs", n)
    t = _all_types_table(n, mask, np.random.default_rng(page_rows))
    path = str(tmp_path / "l.parquet")
    pq.write_table(t, path, data_page_size=1, write_batch_size=page_rows, row_group_size=6_007, data_page_version=page_version, compression="none",
                   use_dictionary=["i64_dict", "dec30_dict"], column_encoding={"b_plain": "PLAIN", "b_rle": "RLE"})
    for name, enc in (("b_rle", RLE), ("i64_dict", RLE_DICTIONARY), ("b_plain", PLAIN)):
        pages = _data_pages(path, 0, t.schema.names.index(name))
        assert {pg["encoding"] for pg in pages} == {enc}, name
    pages = _data_pages(path, 0, t.schema.names.index("b_rle"))
    assert len(pages) == -(-6_007 // page_rows) and {pg["num_values"] for pg in pages[:-1]} == {page_rows}, [pg["num_values"] for pg in pages[:4]]
    assert page_rows == 1000 or _all_null_pages_between_valid(path, t.schema.names.index("b_rle"), mask)
    if page_rows != 1000:
        before = pq.read_table(path)
        assert _poison_level_padding(path, t.schema.names.index("i32")) > 10 and pq.read_table(path).equals(before)
    _check_file(path)


# ---- 5. refusals ---------------------------------------------------------------------------------------------------------
def _refusal_case(kind, x):
    """(table, writer options, the plan's schema, what the metadata must show)"""
    i64 = pa.schema([pa.field("x", pa.int64())])
    ts = pa.schema([pa.field("x", pa.timestamp("us"))])
    if kind == "delta":
        return pa.table({"x": x}), dict(use_dictionary=False, column_encoding={"x": "DELTA_BINARY_PACKED"}), None, ("encoding", "DELTA_BINARY_PACKED")
    if kind == "byte_stream_split":
        return pa.table({"x": x.cast(pa.float64())}), dict(use_dictionary=False, column_encoding={"x": "BYTE_STREAM_SPLIT"}), None, ("encoding", "BYTE_STREAM_SPLIT")
    if kind.startswith("uint"):
        bits = int(kind[4:])
        plan = {8: pa.int8(), 16: pa.int16(), 32: pa.int32(), 64: pa.int64()}[bits]        # the signed type of the same width
        return pa.table({"x": x.cast({8: pa.uint8(), 16: pa.uint16(), 32: pa.uint32(), 64: pa.uint64()}[bits])}), {}, pa.schema([pa.field("x", plan)]), ("logical", f"Int(bitWidth={bits}, isSigned=false)")
    if kind == "ts_millis":
        return pa.table({"x": x.cast(pa.timestamp("ms"))}), {}, ts, ("logical", "Timestamp(isAdjustedToUTC=false, timeUnit=milliseconds")
    if kind == "ts_nanos":
        return pa.table({"x": x.cast(pa.timestamp("ns"))}), {}, ts, ("logical", "Timestamp(isAdjustedToUTC=false, timeUnit=nanoseconds")
    if kind == "int96":
        return pa.table({"x": x.cast(pa.timestamp("ns"))}), dict(use_deprecated_int96_timestamps=True), ts, ("physical", "INT96")
    return pa.table({"x": x}), dict(compression=kind), i64, ("codec", {"gzip": "GZIP", "brotli": "BROTLI", "lz4": "LZ4"}[kind])


@pytest.mark.parametrize("kind", ["delta", "byte_stream_split", "uint8", "uint16", "uint32", "uint64", "ts_millis", "ts_nanos", "int96", "gzip", "brotli", "lz4"])
def test_unsupported_shapes_are_refused(tmp_path, kind):
    x = pa.array(np.arange(1000, dtype=np.int64) % 200)
    t, kw, schema, (what, want) = _refusal_case(kind, x)
    path = str(tmp_path / "r.parquet")
    pq.write_table(t, path, **kw)
    f = pq.ParquetFile(path)
    cc, col = f.metadata.row_group(0).column(0), f.schema.column(0)
    shown = {"encoding": " ".join(cc.encodings), "codec": cc.compression, "physical": col.physical_type, "logical": str(col.logical_type)}[what]
    assert want in shown, (what, shown)
    with pytest.raises(native.NativeError) as ei:
        PL.collect(parquet_scan(path, schema or t.schema))
    assert ei.value.code == native.ERR_UNSUPPORTED, ei.value
    ok = str(tmp_path / "ok.parquet")                             # the refusal leaves nothing behind: the next scan decodes
    pq.write_table(pa.table({"x": x, "y": x.cast(pa.int32())}), ok, compression="snappy")
    _check_file(ok)


# ---- 6. row-group pruning -------------------------------------------------------------------------------------------------
PRUNE_COLS = {"i8": (pa.int8(), T.int8, 8), "i16": (pa.int16(), T.int16, 16), "i32": (pa.int32(), T.int32, 32), "i64": (pa.int64(), T.int64, 64),
              "d": (pa.date32(), T.date32, 32), "ts": (pa.timestamp("us"), T.timestamp_us, 64)}
IGNORED = {"f64": (pa.float64(), T.float64), "dec": (pa.decimal128(12, 2), T.decimal128(12, 2)), "b": (pa.bool_(), T.bool_)}
RG_ROWS, N_RG, NULL_RG = 64, 41, 17


def _prune_table():
    rng = np.random.default_rng(2024)
    n = RG_ROWS * N_RG
    sortedv = lambda lo, hi, dt: np.sort(rng.integers(lo, hi, n, dtype=np.int64)).astype(dt)
    cols = {"i8": sortedv(-128, 128, np.int8), "i16": rng.integers(-2**15, 2**15, n).astype(np.int16),
            "i32": sortedv(-2**31, 2**31, np.int32), "i64": rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True),
            "d": sortedv(-2**31, 2**31, np.int32), "ts": rng.integers(-2**62, 2**62, n, dtype=np.int64)}
    cols["i64"][[5, 900, 2000]] = [I64_MIN, I64_MAX, I64_MIN + 1]
    cols["i16"][[70, 71]] = [-2**15, 2**15 - 1]
    base = rng.random(n) < 0.05
    base[NULL_RG * RG_ROWS: (NULL_RG + 1) * RG_ROWS] = True                    # one row group with nothing but NULLs: no min / max
    arrays = {c: pa.array(v if c != "d" else v, mask=base).cast(PRUNE_COLS[c][0]) for c, v in cols.items()}
    arrays["f64"] = pa.array(rng.normal(size=n) * 100, mask=base)
    arrays["dec"] = pa.array([decimal.Decimal(int(v)).scaleb(-2) for v in rng.integers(-10**6, 10**6, n)], IGNORED["dec"][0], mask=base)
    arrays["b"] = pa.array(np.arange(n) // RG_ROWS % 2 == 0, mask=base)          # constant per row group: min == max
    return pa.table(arrays)


def _stats(md):
    """per row group, per integer-like column: (min, max) as the stored integers, or None when the statistics hold no min / max"""
    out = []
    for g in range(md.num_row_groups):
        row = {}
        for i, name in enumerate(md.schema.names):
            s = md.row_group(g).column(i).statistics
            row[name] = None if s is None or not s.has_min_max else (s.min_raw, s.max_raw)
        out.append(row)
    return out


class _Leaf:
    """`col op lit` or `lit op col`; cast: the column is widened to int64 first (an int64 literal against a narrower column)"""

    def __init__(self, col, op, lit, lit_left, cast=False):
        self.col, self.op, self.lit, self.lit_left, self.cast = col, op, lit, lit_left, cast

    def expr(self):
        if self.col in IGNORED:
            c, lit = E.Column(self.col), E.Literal(self.lit, IGNORED[self.col][1])
        else:
            c = E.Cast(E.Column(self.col), T.int64) if self.cast else E.Column(self.col)
            lit = E.Literal(self.lit, T.int64 if self.cast else PRUNE_COLS[self.col][1])
        return E.BinaryExpr(lit, self.op, c) if self.lit_left else E.BinaryExpr(c, self.op, lit)

    def arrow(self):
        f = pc.field(self.col)
        if self.col in IGNORED:
            ty = IGNORED[self.col][0]
            s = pc.scalar(pa.scalar(decimal.Decimal(self.lit).scaleb(-2) if self.col == "dec" else self.lit, ty))
        elif self.cast:
            f, s = f.cast(pa.int64()), pc.scalar(pa.scalar(self.lit, pa.int64()))
        else:
            ty = PRUNE_COLS[self.col][0]
            s = pc.scalar(pa.scalar(self.lit, pa.int32() if self.col == "d" else pa.int64() if self.col == "ts" else ty).cast(ty))
        a, b = (s, f) if self.lit_left else (f, s)
        return {"Eq": a == b, "NotEq": a != b, "Lt": a < b, "LtEq": a <= b, "Gt": a > b, "GtEq": a >= b}[self.op]

    def may_match(self, stats):
        """can some x in [min, max] satisfy the comparison?  Only a plain column against a literal of its own integer-like type,
        with both statistics present, can answer no"""
        if self.col in IGNORED or self.cast or self.op == "NotEq" or stats[self.col] is None:
            return True
        mn, mx, v = *stats[self.col], self.lit
        if self.lit_left:                                                  # v op x, read as written (not via the mirrored operator)
            return {"Eq": mn <= v <= mx, "Lt": v < mx, "LtEq": v <= mx, "Gt": v > mn, "GtEq": v >= mn}[self.op]
        return {"Eq": mn <= v <= mx, "Lt": mn < v, "LtEq": mn <= v, "Gt": mx > v, "GtEq": mx >= v}[self.op]

    def __repr__(self):
        c = f"cast({self.col})" if self.cast else self.col
        return f"({self.lit} {self.op} {c})" if self.lit_left else f"({c} {self.op} {self.lit})"


class _Node:
    def __init__(self, op, a, b):
        self.op, self.a, self.b = op, a, b

    def expr(self):
        return E.BinaryExpr(self.a.expr(), self.op, self.b.expr())

    def arrow(self):
        return (self.a.arrow() & self.b.arrow()) if self.op == "And" else (self.a.arrow() | self.b.arrow())

    def may_match(self, stats):
        return self.a.may_match(stats) and self.b.may_match(stats) if self.op == "And" else self.a.may_match(stats) or self.b.may_match(stats)

    def __repr__(self):
        return f"({self.a!r} {self.op} {self.b!r})"


def _random_leaf(rng, stats):
    if rng.random() < 0.08:                                                 # a type the pruner must ignore
        col = str(rng.choice(list(IGNORED)))
        lit = {"f64": float(rng.normal() * 100), "dec": int(rng.integers(-10**6, 10**6)), "b": bool(rng.random() < 0.5)}[col]
        return _Leaf(col, str(rng.choice(["Eq", "Lt", "GtEq"])), lit, bool(rng.random() < 0.5))
    col = str(rng.choice(list(PRUNE_COLS)))
    bits = PRUNE_COLS[col][2]
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    cast = col in ("i8", "i16", "i32") and rng.random() < 0.2                # widened to int64 against an int64 literal
    g = stats[int(rng.integers(len(stats)))][col] or (0, 0)
    pick = int(rng.integers(8))
    lit = [g[0], g[1], g[0] - 1, g[1] + 1, lo, hi, I64_MIN, I64_MAX][pick]
    if not cast:
        lit = min(max(lit, lo), hi)                                         # a literal of the column's own type
    op = str(rng.choice(["Eq", "NotEq", "Lt", "LtEq", "Gt", "GtEq"]))
    return _Leaf(col, op, lit, bool(rng.random() < 0.5), cast)


def _random_pred(rng, stats, depth):
    if depth == 0 or rng.random() < 0.4:
        return _random_leaf(rng, stats)
    return _Node(str(rng.choice(["And", "Or"])), _random_pred(rng, stats, depth - 1), _random_pred(rng, stats, depth - 1))


N_PREDICATES = 300


@pytest.fixture(scope="module")
def prune_file(tmp_path_factory):
    t = _prune_table()
    path = str(tmp_path_factory.mktemp("prune") / "p.parquet")
    pq.write_table(t, path, row_group_size=RG_ROWS, compression="snappy", use_dictionary=["i16", "b"])
    md = pq.ParquetFile(path).metadata
    assert md.num_row_groups == N_RG
    stats = _stats(md)
    assert all(stats[NULL_RG][c] is None for c in t.schema.names) and all(stats[g]["i32"] is not None for g in range(N_RG) if g != NULL_RG)
    return path, t.schema, md, stats


@pytest.mark.parametrize("seed", range(100, 100 + N_PREDICATES // 25), ids=lambda s: f"seed{s}")
def test_pruning_is_sound_and_exact(prune_file, seed):
    """(a) FilterExec over the pruned scan returns pyarrow's filter of the same predicate; (b) the scan alone keeps exactly the row
    groups an independent reading of the statistics keeps (input_batches = row groups decoded): the pruner can neither lose rows
    nor be silently disabled"""
    path, schema, md, stats = prune_file
    rng = np.random.default_rng(seed)
    table = pq.read_table(path)
    pruned_total = 0
    for i in range(25):
        pred = _random_pred(rng, stats, 3)
        e = pred.expr()
        out = PL.collect(PL.FilterExec([e], parquet_scan(path, schema, pruning_predicates=[e])))
        assert_same_table(out, table.filter(pred.arrow()))
        keep = [pred.may_match(s) for s in stats]
        _, m = _scan_all(path, schema, projection=[0], pruning_predicates=[e])
        assert m["input_batches"] == sum(keep), (pred, m["input_batches"], sum(keep))
        pruned_total += N_RG - sum(keep)
    assert pruned_total > 25 * N_RG // 10, pruned_total                # the predicates do prune: not a vacuous check


@pytest.mark.parametrize("splits", [3, 7])
def test_pruning_with_split_ranges(prune_file, splits):
    """with the file cut into byte ranges, every kept row group is decoded by exactly the split holding its first byte"""
    path, schema, md, stats = prune_file
    size = os.path.getsize(path)
    cuts = [size * i // splits for i in range(splits + 1)]
    first = []
    for g in range(N_RG):
        cc = md.row_group(g).column(0)
        first.append(min(cc.data_page_offset, cc.dictionary_page_offset) if cc.has_dictionary_page else cc.data_page_offset)
    assert len({sum(c <= f for c in cuts[1:-1]) for f in first}) >= splits - 1, "splits without row groups"     # the last may hold only the footer
    table = pq.read_table(path)
    rng = np.random.default_rng(splits)
    for _ in range(25):
        pred = _random_pred(rng, stats, 2)
        e = pred.expr()
        keep = [pred.may_match(s) for s in stats]
        outs = []
        for lo, hi in zip(cuts, cuts[1:]):
            _, m = _scan_all(path, schema, projection=[0], pruning_predicates=[e], range=(lo, hi))
            assert m["input_batches"] == sum(k for k, f in zip(keep, first) if lo <= f < hi), (pred, lo, hi)
            outs += PL.collect(PL.FilterExec([e], parquet_scan(path, schema, pruning_predicates=[e], range=(lo, hi))))
        assert_same_table(outs, table.filter(pred.arrow()))
