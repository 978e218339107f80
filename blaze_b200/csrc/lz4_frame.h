// LZ4 frame encoder and decoder (lz4_frame.cc): the compression blocks of the shuffle files.
#pragma once
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200q {

uint32_t xxhash32(const uint8_t* p, size_t n, uint32_t seed);
size_t lz4_block_bound(size_t n);
size_t lz4_block_compress(const uint8_t* src, size_t n, uint8_t* dst);          // dst holds lz4_block_bound(n) bytes
void lz4_frame_append(const uint8_t* src, size_t n, std::vector<uint8_t>& out);  // one complete frame appended to `out`

// A frame that breaks the format: `offset` is the byte of the input where the decoder stopped.
struct Lz4FrameError : std::runtime_error {
  size_t offset;
  Lz4FrameError(const std::string& m, size_t off) : std::runtime_error(m), offset(off) {}
};
// src[0, n) holds one or more concatenated LZ4 frames.  lz4_frame_bound walks their headers and block sizes only and returns
// an upper bound of the decoded size (exact when every frame declares its content size); lz4_frame_decompress decodes them into
// dst (capacity cap) and returns the decoded size.  Both throw Lz4FrameError on anything the format does not allow; the decoder
// never reads outside src[0, n) nor writes outside dst[0, cap).
size_t lz4_frame_bound(const uint8_t* src, size_t n);
size_t lz4_frame_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap);

}  // namespace b200q
