"""LZ4 frames of every shape the frame format allows, built around liblz4 (pyarrow) for the tests of the library's decoder.

pyarrow's "lz4" codec writes one shape only (linked 64 KiB blocks, no checksums, no content size); "lz4_raw" compresses one
independent block.  `reframe` re-emits the blocks of a pyarrow frame under other header flags, `frame` builds a frame of
independent blocks of any maximum size.  xxh32 follows the xxHash specification (it is what the frame checksums use)."""
import struct

import pyarrow as pa

_P1, _P2, _P3, _P4, _P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
_M = 0xFFFFFFFF
BLOCK_MAX = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}


def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & _M


def xxh32(data: bytes, seed: int = 0) -> int:
    n, p = len(data), 0
    if n >= 16:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed & _M, (seed - _P1) & _M]
        words = struct.unpack_from("<%dI" % ((n // 16) * 4), data)
        for i in range(0, len(words), 4):
            for k in range(4):
                v[k] = (_rotl((v[k] + words[i + k] * _P2) & _M, 13) * _P1) & _M
        p = (n // 16) * 16
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while p + 4 <= n:
        h = (_rotl((h + struct.unpack_from("<I", data, p)[0] * _P3) & _M, 17) * _P4) & _M
        p += 4
    while p < n:
        h = (_rotl((h + data[p] * _P5) & _M, 11) * _P1) & _M
        p += 1
    h ^= h >> 15; h = (h * _P2) & _M; h ^= h >> 13; h = (h * _P3) & _M; h ^= h >> 16
    return h


def header(bs_code: int, independent: bool, block_cksum: bool, content_size, content_cksum: bool) -> bytes:
    flg = 0x40 | (0x20 if independent else 0) | (0x10 if block_cksum else 0) | (0x08 if content_size is not None else 0) | (0x04 if content_cksum else 0)
    desc = bytes([flg, bs_code << 4]) + (struct.pack("<Q", content_size) if content_size is not None else b"")
    return struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32(desc) >> 8) & 0xFF])


def _emit(blocks, content: bytes, bs_code, independent, block_cksum, with_size, content_cksum) -> bytes:
    out = bytearray(header(bs_code, independent, block_cksum, len(content) if with_size else None, content_cksum))
    for payload, stored in blocks:
        out += struct.pack("<I", len(payload) | (0x80000000 if stored else 0)) + payload
        if block_cksum:
            out += struct.pack("<I", xxh32(payload))
    out += b"\0\0\0\0"
    if content_cksum:
        out += struct.pack("<I", xxh32(content))
    return bytes(out)


def pyarrow_blocks(fr: bytes):
    """(payload, stored) of every data block of a frame pyarrow wrote (its header: 7 bytes, no optional fields)"""
    pos, out = 7, []
    while True:
        (w,) = struct.unpack_from("<I", fr, pos); pos += 4
        if w == 0:
            return out
        n = w & 0x7FFFFFFF
        out.append((fr[pos: pos + n], bool(w >> 31))); pos += n


def reframe(data: bytes, bs_code=4, block_cksum=False, with_size=False, content_cksum=False) -> bytes:
    """liblz4's linked blocks (of 64 KiB) of `data` under another header"""
    fr = pa.Codec("lz4").compress(data, asbytes=True)
    blocks = pyarrow_blocks(fr)
    assert all(len(p) <= BLOCK_MAX[bs_code] for p, _ in blocks), "pyarrow's frame shape changed"
    return _emit(blocks, data, bs_code, bool(fr[4] & 0x20), block_cksum, with_size, content_cksum)      # a one-block frame says independent


def frame(data: bytes, bs_code=7, block_cksum=False, with_size=False, content_cksum=False, stored_every=0) -> bytes:
    """independent blocks of BLOCK_MAX[bs_code] bytes, each compressed by liblz4's block compressor (or stored: every
    `stored_every`-th block, and any block that does not shrink)"""
    c, bm, blocks = pa.Codec("lz4_raw"), BLOCK_MAX[bs_code], []
    for i, p in enumerate(range(0, len(data), bm)):
        chunk = data[p: p + bm]
        z = c.compress(chunk, asbytes=True)
        stored = (stored_every and i % stored_every == 0) or len(z) >= len(chunk)
        blocks.append((chunk, True) if stored else (z, False))
    return _emit(blocks, data, bs_code, True, block_cksum, with_size, content_cksum)
