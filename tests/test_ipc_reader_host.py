"""IpcReaderExec without a GPU: decoding and explaining the IpcReaderExecNode leaf and its refusals, and the library's LZ4 frame
decoder (b200q_lz4_frame_decompress) against frames from liblz4 (pyarrow) and from the library's own encoder, and against every
way a frame can break the format."""
import ctypes as C
import struct

import numpy as np
import pyarrow as pa
import pytest

import lz4_frames as LF
from blaze_b200 import exprs as E, native, plans as PL, proto as P, types as T
from blaze_b200.types import Field, Schema

ALL_TYPES = [("i8", T.int8), ("i16", T.int16), ("i32", T.int32), ("i64", T.int64), ("f32", T.float32), ("f64", T.float64),
             ("d", T.date32), ("ts", T.timestamp_us), ("dec", T.decimal128(38, 4)), ("b", T.bool_), ("bin", T.binary), ("s", T.utf8)]


def _status(fn):
    with pytest.raises(native.NativeError) as ei:
        fn()
    return ei.value


# ---- plan decode / explain -------------------------------------------------------------------------------------------------
def test_explain_every_supported_type():
    s = Schema([Field(n, t, i % 2 == 0) for i, (n, t) in enumerate(ALL_TYPES)])
    text = PL.IpcReaderExec(s, resource_id="shuffle-3").explain()
    assert text.startswith("IpcReader schema=[i8:int8?, i16:int16, ")
    assert "dec:decimal128(38,4)?" in text and "bin:binary?" in text and "s:utf8]" in text


def test_node_wire_form():
    s = Schema([Field("k", T.int64, False)])
    node = P.PhysicalPlanNode()
    node.ParseFromString(PL.IpcReaderExec(s, num_partitions=200, resource_id="rid").plan_bytes())
    assert node.WhichOneof("PhysicalPlanType") == "ipc_reader"
    assert (node.ipc_reader.num_partitions, node.ipc_reader.ipc_provider_resource_id) == (200, "rid")
    assert node.SerializeToString()[:1] == b"\x1a"                      # field 3, wire type 2


def test_reduce_plans_over_the_leaf_decode():
    ins = Schema([Field("k", T.int64, False), Field(E.AGG_BUF_COLUMN_NAME, T.binary, False)])
    leaf = PL.IpcReaderExec(ins)
    final = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))],
                       [E.AggExpr("s", E.FINAL, PL.create_agg(E.AGG_SUM, [E.placeholder(T.int64)], ins, T.int64))], False, leaf)
    top = PL.SortExec(final, [(E.Column("s"), True, False)], fetch=10)
    text = top.explain()
    assert "SortExec" in text and "AggExec" in text and text.splitlines()[-1].strip().startswith("IpcReader schema=[k:int64")


def _raw_field(name: bytes, arrow_type: bytes) -> bytes:
    f = b"\x0a" + bytes([len(name)]) + name + b"\x12" + bytes([len(arrow_type)]) + arrow_type
    return b"\x0a" + bytes([len(f)]) + f                               # Schema.columns = 1


def _raw_ipc_node(schema: bytes) -> bytes:
    body = b"\x08\x01" + (b"\x12" + bytes([len(schema)]) + schema if schema is not None else b"")
    return b"\x1a" + bytes([len(body)]) + body


def test_missing_schema_is_invalid_plan():
    e = _status(lambda: native.plan_explain(_raw_ipc_node(None)))
    assert e.code == native.ERR_INVALID_PLAN and "leaf node without schema" in e.msg


def test_null_column_is_unsupported():
    e = _status(lambda: native.plan_explain(_raw_ipc_node(_raw_field(b"nothing", b"\x0a\x00"))))   # ArrowType.NONE
    assert e.code == native.ERR_UNSUPPORTED and "nothing" in e.msg and "Null" in e.msg


@pytest.mark.parametrize("tag", [3, 32, 26])                             # UINT8, LargeUtf8, a type outside the hot path
def test_other_types_are_unsupported_with_the_column_name(tag):
    e = _status(lambda: native.plan_explain(_raw_ipc_node(_raw_field(b"colx", bytes([(tag << 3) | 2, 0]) if tag < 16 else bytes([((tag << 3) | 2) & 0x7F | 0x80, (tag << 3) >> 7, 0])))))
    assert e.code == native.ERR_UNSUPPORTED and "colx" in e.msg


# ---- LZ4 frame decoder -------------------------------------------------------------------------------------------------------
def _data(kind: str, n: int) -> bytes:
    rng = np.random.default_rng(n)
    if kind == "planes":
        return np.frombuffer(rng.integers(-10**6, 10**6, n // 8, dtype=np.int64).tobytes(), np.uint8).reshape(-1, 8).T.tobytes()
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    return (b"the quick brown fox jumps over the lazy dog " * (n // 44 + 1))[:n]


@pytest.mark.parametrize("n", [0, 1, 13, 70_000, 300_000])
@pytest.mark.parametrize("kind", ["planes", "random", "text"])
def test_pyarrow_frames(kind, n):
    d = _data(kind, n)
    assert native.lz4_frame_decompress(pa.Codec("lz4").compress(d, asbytes=True)) == d


@pytest.mark.parametrize("bs", [4, 5, 6, 7])
@pytest.mark.parametrize("linked", [True, False])
@pytest.mark.parametrize("flags", ["none", "size", "block_ck", "content_ck", "all"])
def test_every_frame_shape(bs, linked, flags):
    d = _data("planes", 3 * LF.BLOCK_MAX[bs] // 2 + 777 if bs < 7 else 600_000)
    kw = dict(with_size=flags in ("size", "all"), block_cksum=flags in ("block_ck", "all"), content_cksum=flags in ("content_ck", "all"))
    fr = LF.reframe(d, bs, **kw) if linked else LF.frame(d, bs, **kw)
    assert native.lz4_frame_decompress(fr) == d


def test_stored_blocks_and_concatenated_frames():
    d = _data("planes", 200_000)
    fr = LF.frame(d, 4, stored_every=2, block_cksum=True)
    assert native.lz4_frame_decompress(fr) == d
    assert native.lz4_frame_decompress(fr + LF.reframe(d[:1000], 5)) == d + d[:1000]
    assert native.lz4_frame_decompress(LF.frame(_data("random", 100_000), 4)) == _data("random", 100_000)   # incompressible: stored


@pytest.mark.parametrize("name", ["empty", "one byte", "twelve bytes", "thirteen bytes", "text", "random", "byte planes", "zeros above one block", "random above one block"])
def test_frames_of_the_library_encoder(name):
    rng = np.random.default_rng(7)                                       # the inputs of tests/test_lz4_frame.py
    data = {"empty": b"", "one byte": b"x", "twelve bytes": b"abcabcabcabc", "thirteen bytes": b"abcabcabcabca", "text": b"the quick brown fox " * 5000,
            "random": rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes(),
            "byte planes": np.frombuffer(rng.integers(-10**6, 10**6, 100_000, dtype=np.int64).tobytes(), np.uint8).reshape(-1, 8).T.tobytes(),
            "zeros above one block": bytes(9 << 20), "random above one block": rng.integers(0, 256, (4 << 20) + 12345, dtype=np.uint8).tobytes()}[name]
    assert native.lz4_frame_decompress(native.lz4_frame_compress(data)) == data


def test_too_small_output_buffer_reports_the_size():
    fr = native.lz4_frame_compress(b"hello world, hello world, hello world")
    need = C.c_size_t(0)
    buf = C.create_string_buffer(4)
    assert native.lib.b200q_lz4_frame_decompress(fr, len(fr), buf, 4, C.byref(need)) == native.ERR_INVALID_ARG
    assert need.value == 37 and "needs 37 bytes" in native.last_error()


def _block_frame(block: bytes, bs=4) -> bytes:
    return LF.header(bs, True, False, None, False) + struct.pack("<I", len(block)) + block + b"\0\0\0\0"


def _with_hc(fr: bytes) -> bytes:
    """the header checksum recomputed after editing the descriptor (FLG, BD, content size)"""
    end = 6 + (8 if fr[4] & 0x08 else 0)
    return fr[:end] + bytes([(LF.xxh32(fr[4:end]) >> 8) & 0xFF]) + fr[end + 1:]


def _malformed():
    good = LF.frame(_data("planes", 100_000), 4, block_cksum=True, with_size=True, content_cksum=True)
    hc = 4 + 2 + 8                                                       # magic, FLG BD, content size
    long_match = bytes([0x1F]) + b"a" + b"\x01\x00" + b"\xff" * 275 + b"\x00" + bytes([0x10]) + b"b"   # 'a' x ~70 KB > 64 KiB block
    return {
        "empty input": b"",
        "bad magic": b"\x05" + good[1:],
        "zstd magic": bytes([0x28, 0xB5, 0x2F, 0xFD]) + good[4:],
        "version 00": _with_hc(good[:4] + bytes([good[4] & 0x3F]) + good[5:]),
        "reserved FLG bit": _with_hc(good[:4] + bytes([good[4] | 0x02]) + good[5:]),
        "dictionary id": _with_hc(good[:4] + bytes([good[4] | 0x01]) + good[5:]),
        "reserved BD bit": _with_hc(good[:5] + bytes([good[5] | 0x80]) + good[6:]),
        "reserved BD code": _with_hc(good[:5] + bytes([0x30]) + good[6:]),
        "header checksum": good[:hc] + bytes([good[hc] ^ 1]) + good[hc + 1:],
        "truncated header": good[:9],
        "truncated block": good[: len(good) // 2],
        "missing end mark": good[:-8],
        "block above the maximum": LF.header(4, True, False, None, False) + struct.pack("<I", (64 << 10) + 1) + bytes((64 << 10) + 1) + b"\0" * 4,
        "match before the output start": _block_frame(bytes([0x04]) + b"\x05\x00" + bytes([0x10]) + b"z"),
        "zero match offset": _block_frame(bytes([0x14]) + b"q\x00\x00" + bytes([0x10]) + b"z"),
        "literals past the block": _block_frame(bytes([0x50]) + b"ab"),
        "truncated match offset": _block_frame(bytes([0x14]) + b"q\x01"),
        "output overrun": _block_frame(long_match),
        "block checksum": good[:-12] + bytes([good[-12] ^ 0xFF]) + good[-11:],
        "content checksum": good[:-1] + bytes([good[-1] ^ 0xFF]),
        "content size": _with_hc(good[:6] + struct.pack("<Q", 99_999) + good[14:]),
        "trailing garbage": good + b"\x01\x02",
    }


@pytest.mark.parametrize("name", list(_malformed()))
def test_malformed_frames_are_invalid_arg(name):
    fr = _malformed()[name]
    e = _status(lambda: native.lz4_frame_decompress(fr))
    assert e.code == native.ERR_INVALID_ARG and "at byte" in e.msg, e.msg


def test_the_long_match_itself_decodes_when_the_block_may_hold_it():
    long_match = bytes([0x1F]) + b"a" + b"\x01\x00" + b"\xff" * 275 + b"\x00" + bytes([0x10]) + b"b"
    out = native.lz4_frame_decompress(_block_frame(long_match, bs=5))
    assert out == b"a" * (1 + 19 + 275 * 255) + b"b"
