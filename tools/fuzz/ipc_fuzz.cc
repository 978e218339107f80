// ASan/UBSan fuzz harness of the reduce side's host decoders: the LZ4 frame decoder (lz4_frame.cc) and the batch_serde record walker
// (ipc_records.cc).  Reads seed files, mutates, decodes.  Every outcome must be a value or an Lz4FrameError / IpcRecordError —
// never a crash, an out-of-bounds access or undefined behaviour.
//   usage: ipc_fuzz <seed> <iterations> --lz4|--records <seed files...>
//   --records seeds: [ncols u8][type id u8 x ncols][stream bytes]; the stream is split into 1-4 segments at random points
//   build: see tools/fuzz/run.sh
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <random>
#include <string>
#include <vector>
#include "ipc_records.h"
#include "lz4_frame.h"
using namespace b200q;
int main(int argc, char** argv) {
  std::vector<std::vector<uint8_t>> seeds;
  bool lz4 = std::string(argv[3]) == "--lz4";
  for (int i = 4; i < argc; i++) { std::ifstream f(argv[i], std::ios::binary); seeds.emplace_back(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>()); }
  std::mt19937_64 rng(atoll(argv[1])); long n = atol(argv[2]); long ok = 0, err = 0;
  std::vector<uint8_t> out;
  for (long it = 0; it < n; it++) {
    std::vector<uint8_t> b = seeds[rng() % seeds.size()];
    const int k = rng() % 10;
    if (k < 4) { for (int j = 0, m = 1 + rng() % 4; j < m; j++) b[rng() % b.size()] = (uint8_t)rng(); }
    else if (k < 6) b.resize(rng() % b.size());
    if (b.empty()) b.push_back(0);
    else if (k < 8) { size_t i = rng() % b.size(), j = std::min(b.size(), i + 1 + rng() % 16); b.erase(b.begin() + i, b.begin() + j); }
    else if (k < 9) { size_t i = rng() % b.size(); for (int j = 0, m = 1 + rng() % 8; j < m; j++) b.insert(b.begin() + i, (uint8_t)rng()); }
    try {
      if (lz4) {
        const size_t bound = lz4_frame_bound(b.data(), b.size());
        out.resize(std::min<size_t>(bound, (size_t)64 << 20) + 1);
        ok += lz4_frame_decompress(b.data(), b.size(), out.data(), std::min<size_t>(bound, (size_t)64 << 20)) <= bound;
      } else {
        const size_t nc = b[0] % 8;
        if (b.size() < 1 + nc) { err++; continue; }
        std::vector<DType> types(nc);
        for (size_t c = 0; c < nc; c++) { types[c].id = (TypeId)(b[1 + c] % (T_UTF8 + 1)); if (types[c].id == T_NULL) types[c].id = T_INT64; }
        std::vector<uint8_t> body(b.begin() + 1 + (ptrdiff_t)nc, b.end());
        std::vector<std::vector<uint8_t>> parts;                   // separate allocations: a read across a segment end is caught
        std::vector<IpcSegment> segs;
        size_t pos = 0;
        for (int s = 0, ns = 1 + (int)(rng() % 4); s < ns; s++) {
          const size_t take = s + 1 == ns ? body.size() - pos : (body.size() - pos ? rng() % (body.size() - pos + 1) : 0);
          parts.emplace_back(body.begin() + (ptrdiff_t)pos, body.begin() + (ptrdiff_t)(pos + take)); pos += take;
        }
        for (auto& p : parts) segs.push_back(IpcSegment{p.data(), p.size()});
        IpcRecordTable t; t.ncols = nc;
        ipc_walk_records(segs, types, t);
        ok += (long)t.count() >= 0;
      }
    } catch (const std::exception&) { err++; }
  }
  printf("%s ok=%ld err=%ld\n", lz4 ? "lz4_frame" : "ipc_records", ok, err);
}
