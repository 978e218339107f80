// LZ4 frame encoder of the shuffle files' compression blocks (host side; the GPU produces the uncompressed batch_serde bytes),
// and the decoder of the reduce side (IpcReaderExec, ipc_source.cu), written from the same specifications.
//
// The reference frames every shuffle block as `u32 LE length ‖ LZ4 frame` with lz4_flex's FrameEncoder
// (datafusion-ext-plans/src/common/ipc_compression.rs:34-112, codec "lz4" = spark.io.compression.codec default :271-283).
// lz4_flex is not vendored; what is restated here is the published LZ4 Frame Format 1.6.x and Block Format: magic
// 0x184D2204, FLG (version 01, independent blocks, no checksums, no content size), BD (4 MiB blocks), HC = second byte of
// xxHash32(descriptor, 0); data blocks `u32 size (bit 31 = stored) ‖ bytes`; EndMark 0.  Any conforming decoder
// (lz4_flex's FrameDecoder, liblz4's LZ4F_decompress via pyarrow in the tests) reads it.  The block compressor is a
// single-pass greedy matcher (64 Ki-entry hash table of 4-byte sequences, 64 KiB window): the byte-plane layout of
// batch_serde makes long runs of equal high-order bytes, which this finds as RLE-style matches.
#include "lz4_frame.h"

#include <algorithm>
#include <cstring>

namespace b200q {

namespace {

inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
inline uint32_t rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

constexpr uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;

}  // namespace

uint32_t xxhash32(const uint8_t* p, size_t n, uint32_t seed) {
  const uint8_t* end = p + n;
  uint32_t h;
  if (n >= 16) {
    uint32_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
    do {
      v1 = rotl(v1 + rd32(p) * P2, 13) * P1; v2 = rotl(v2 + rd32(p + 4) * P2, 13) * P1;
      v3 = rotl(v3 + rd32(p + 8) * P2, 13) * P1; v4 = rotl(v4 + rd32(p + 12) * P2, 13) * P1;
      p += 16;
    } while (p + 16 <= end);
    h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
  } else h = seed + P5;
  h += (uint32_t)n;
  while (p + 4 <= end) { h = rotl(h + rd32(p) * P3, 17) * P4; p += 4; }
  while (p < end) { h = rotl(h + (*p) * P5, 11) * P1; p++; }
  h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
  return h;
}

size_t lz4_block_bound(size_t n) { return n + n / 255 + 16; }

// LZ4 block format: sequences of [token][literal length bytes][literals][offset u16 LE][match length bytes]; the last
// sequence has literals only; the last 5 bytes are literals and no match starts within the last 12 bytes.
size_t lz4_block_compress(const uint8_t* src, size_t n, uint8_t* dst) {
  constexpr int HBITS = 16;
  static thread_local uint32_t table[1 << HBITS];
  uint8_t* op = dst;
  size_t anchor = 0;
  auto emit_literals_and_match = [&](size_t lit_len, const uint8_t* lit, bool has_match, size_t offset, size_t mlen) {
    uint8_t* token = op++;
    size_t l = lit_len;
    if (l >= 15) { *token = 0xF0; l -= 15; while (l >= 255) { *op++ = 255; l -= 255; } *op++ = (uint8_t)l; } else *token = (uint8_t)(l << 4);
    memcpy(op, lit, lit_len); op += lit_len;
    if (!has_match) return;
    *op++ = (uint8_t)offset; *op++ = (uint8_t)(offset >> 8);
    size_t m = mlen - 4;
    if (m >= 15) { *token |= 15; m -= 15; while (m >= 255) { *op++ = 255; m -= 255; } *op++ = (uint8_t)m; } else *token |= (uint8_t)m;
  };
  if (n >= 13) {
    memset(table, 0, sizeof(table));                                  // positions are stored + 1 (0 = empty)
    const size_t mflimit = n - 12, matchlimit = n - 5;
    size_t ip = 0, misses = 0;
    while (ip < mflimit) {
      const uint32_t seq = rd32(src + ip);
      const uint32_t h = (seq * 2654435761u) >> (32 - HBITS);
      const size_t ref = table[h];
      table[h] = (uint32_t)(ip + 1);
      if (ref && ip + 1 - ref <= 65535 && rd32(src + ref - 1) == seq) {
        const size_t r = ref - 1;
        size_t m = 4;
        while (ip + m + 8 <= matchlimit && rd64(src + ip + m) == rd64(src + r + m)) m += 8;
        while (ip + m < matchlimit && src[ip + m] == src[r + m]) m++;
        emit_literals_and_match(ip - anchor, src + anchor, true, ip - r, m);
        ip += m; anchor = ip; misses = 0;
      } else {
        ip += 1 + (misses++ >> 6);                                    // skip faster through incompressible data
      }
    }
  }
  emit_literals_and_match(n - anchor, src + anchor, false, 0, 0);
  return (size_t)(op - dst);
}

void lz4_frame_append(const uint8_t* src, size_t n, std::vector<uint8_t>& out) {
  constexpr size_t BLOCK = 4u << 20;
  const uint8_t desc[2] = {0x60, 0x70};                               // FLG: version 01, block independence; BD: 4 MiB
  const uint8_t hdr[7] = {0x04, 0x22, 0x4D, 0x18, desc[0], desc[1], (uint8_t)(xxhash32(desc, 2, 0) >> 8)};
  out.insert(out.end(), hdr, hdr + 7);
  for (size_t pos = 0; pos < n; pos += BLOCK) {
    const size_t len = n - pos < BLOCK ? n - pos : BLOCK;
    const size_t at = out.size();
    out.resize(at + 4 + lz4_block_bound(len));
    size_t clen = lz4_block_compress(src + pos, len, out.data() + at + 4);
    uint32_t word;
    if (clen >= len) { memcpy(out.data() + at + 4, src + pos, len); clen = len; word = (uint32_t)len | 0x80000000u; }     // stored block
    else word = (uint32_t)clen;
    memcpy(out.data() + at, &word, 4);
    out.resize(at + 4 + clen);
  }
  const uint8_t endmark[4] = {0, 0, 0, 0};
  out.insert(out.end(), endmark, endmark + 4);
}

// ---- decoder (the reduce side reads what lz4_flex's FrameEncoder, liblz4 or lz4_frame_append wrote) ----------------------
// Frame: magic ‖ FLG ‖ BD ‖ [content size u64] ‖ [dict id u32] ‖ HC, then blocks `u32 size (bit 31 = stored) ‖ bytes ‖
// [xxh32 of the bytes]` up to the EndMark 0, then [xxh32 of the content].  FLG: version 01 (bits 7-6), block independence (5),
// block checksum (4), content size (3), content checksum (2), reserved 0 (1), dict id (0).  BD: reserved 0 (7, 3-0), block
// maximum size 4..7 = 64 KiB..4 MiB (6-4).  Preset dictionaries are not used by any shuffle writer and are refused.

namespace {

struct FrameHeader { bool indep, block_cksum, content_cksum, has_size; uint64_t content_size; size_t block_max, len; };

FrameHeader parse_header(const uint8_t* p, size_t n, size_t base) {
  if (n < 4) throw Lz4FrameError("lz4 frame: truncated magic number", base + n);
  if (rd32(p) != 0x184D2204u) throw Lz4FrameError("lz4 frame: bad magic number", base);
  if (n < 7) throw Lz4FrameError("lz4 frame: truncated frame descriptor", base + n);
  const uint8_t flg = p[4], bd = p[5];
  if ((flg >> 6) != 1) throw Lz4FrameError("lz4 frame: version " + std::to_string(flg >> 6) + " in FLG, only 01 exists", base + 4);
  if (flg & 0x02) throw Lz4FrameError("lz4 frame: reserved FLG bit set", base + 4);
  if (flg & 0x01) throw Lz4FrameError("lz4 frame: preset dictionaries are not supported", base + 4);
  if (bd & 0x8F) throw Lz4FrameError("lz4 frame: reserved BD bits set", base + 5);
  const int bs = (bd >> 4) & 7;
  if (bs < 4) throw Lz4FrameError("lz4 frame: block maximum size code " + std::to_string(bs) + " is reserved", base + 5);
  FrameHeader h;
  h.indep = flg & 0x20; h.block_cksum = flg & 0x10; h.has_size = flg & 0x08; h.content_cksum = flg & 0x04;
  h.block_max = (size_t)1 << (8 + 2 * bs);
  h.content_size = 0;
  size_t len = 6;
  if (h.has_size) {
    if (n < len + 8 + 1) throw Lz4FrameError("lz4 frame: truncated frame descriptor", base + n);
    h.content_size = rd64(p + 6); len += 8;
  }
  if (p[len] != (uint8_t)(xxhash32(p + 4, len - 4, 0) >> 8)) throw Lz4FrameError("lz4 frame: header checksum mismatch", base + len);
  h.len = len + 1;
  return h;
}

// one compressed block s[0, n) appended at dst[o]; a match may reach back to dst[lower] (the frame's start, or the block's for
// independent blocks)
size_t decode_block(const uint8_t* s, size_t n, uint8_t* dst, size_t o, size_t cap, size_t lower, size_t base) {
  size_t i = 0;
  for (;;) {
    if (i >= n) throw Lz4FrameError("lz4 block: truncated sequence", base + i);
    const unsigned tok = s[i++];
    size_t lit = tok >> 4;
    if (lit == 15) {
      unsigned b;
      do { if (i >= n) throw Lz4FrameError("lz4 block: truncated literal length", base + i); b = s[i++]; lit += b; } while (b == 255);
    }
    if (lit > n - i) throw Lz4FrameError("lz4 block: literals run past the end of the block", base + i);
    if (lit > cap - o) throw Lz4FrameError("lz4 block: output overrun", base + i);
    memcpy(dst + o, s + i, lit); i += lit; o += lit;
    if (i == n) return o;                                             // the last sequence holds literals only
    if (n - i < 2) throw Lz4FrameError("lz4 block: truncated match offset", base + i);
    const size_t off = (size_t)s[i] | ((size_t)s[i + 1] << 8);
    if (off == 0 || off > o - lower) throw Lz4FrameError("lz4 block: match offset " + std::to_string(off) + " before the start of the output", base + i);
    i += 2;
    size_t m = (tok & 15) + 4;
    if ((tok & 15) == 15) {
      unsigned b;
      do { if (i >= n) throw Lz4FrameError("lz4 block: truncated match length", base + i); b = s[i++]; m += b; } while (b == 255);
    }
    if (m > cap - o) throw Lz4FrameError("lz4 block: output overrun", base + i);
    const uint8_t* from = dst + o - off;
    if (off >= m) { memcpy(dst + o, from, m); o += m; continue; }
    while (m) {                                                       // overlapping: the pattern of period `off` doubles per copy
      const size_t k = std::min(m, (size_t)(dst + o - from));
      memcpy(dst + o, from, k); o += k; m -= k;
    }
  }
}

// walks (and in decode mode, decodes) every frame of src[0, n)
size_t walk_frames(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, bool decode) {
  size_t pos = 0, out = 0;
  do {
    const FrameHeader h = parse_header(src + pos, n - pos, pos);
    pos += h.len;
    const size_t start = out;
    uint64_t bound = 0;
    for (;;) {
      if (n - pos < 4) throw Lz4FrameError("lz4 frame: truncated block size", n);
      const uint32_t w = rd32(src + pos);
      if (w == 0) { pos += 4; break; }                                  // EndMark
      const size_t sz = w & 0x7FFFFFFFu;
      const bool stored = w >> 31;
      if (sz > h.block_max) throw Lz4FrameError("lz4 frame: block of " + std::to_string(sz) + " bytes above the frame's maximum of " + std::to_string(h.block_max), pos);
      pos += 4;
      const size_t ck = h.block_cksum ? 4 : 0;
      if (n - pos < sz + ck) throw Lz4FrameError("lz4 frame: truncated block", n);
      if (decode) {
        if (stored) {
          if (sz > cap - out) throw Lz4FrameError("lz4 frame: output overrun", pos);
          memcpy(dst + out, src + pos, sz); out += sz;
        } else {
          out = decode_block(src + pos, sz, dst, out, cap, h.indep ? out : start, pos);
        }
        if (ck && rd32(src + pos + sz) != xxhash32(src + pos, sz, 0)) throw Lz4FrameError("lz4 frame: block checksum mismatch", pos + sz);
      }
      bound += stored ? sz : std::min<uint64_t>(h.block_max, (uint64_t)sz * 255);
      pos += sz + ck;
    }
    if (h.content_cksum) {
      if (n - pos < 4) throw Lz4FrameError("lz4 frame: truncated content checksum", n);
      if (decode && rd32(src + pos) != xxhash32(dst + start, out - start, 0)) throw Lz4FrameError("lz4 frame: content checksum mismatch", pos);
      pos += 4;
    }
    if (decode) {
      if (h.has_size && out - start != h.content_size)
        throw Lz4FrameError("lz4 frame: " + std::to_string(out - start) + " bytes decoded, the header declares " + std::to_string(h.content_size), pos);
    } else {
      out += (size_t)(h.has_size ? std::min<uint64_t>(h.content_size, bound) : bound);
    }
  } while (pos < n);
  return out;
}

}  // namespace

size_t lz4_frame_bound(const uint8_t* src, size_t n) { return walk_frames(src, n, nullptr, 0, false); }
size_t lz4_frame_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap) { return walk_frames(src, n, dst, cap, true); }

}  // namespace b200q
