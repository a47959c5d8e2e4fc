// What esvo::PoseBuffer (include/esvo_b200/esvo_system.hpp, the tf buffer of the nodes) answers, for a comparison with the
// Python restatement (tests/test_system_loop.py).  Host logic only: builds with plain g++, no library, no GPU.
// usage: pose_buffer_dump <in.bin> <out.bin>
// in:  i32 n; i64 stamps[n]; f64 poses[n*16] (inserted in this order); i32 m; i64 queries[m]
// out: per query i32 found; f64 T[16] (zeros when not found); then i32 number of stored entries
#include <cstdio>
#include <fstream>

#include "esvo_b200/esvo_system.hpp"

int main(int argc, char** argv) {
  if (argc < 3) { std::printf("usage: pose_buffer_dump <in.bin> <out.bin>\n"); return 64; }
  std::ifstream f(argv[1], std::ios::binary);
  int32_t n = 0, m = 0;
  f.read((char*)&n, 4);
  std::vector<int64_t> st(n); std::vector<double> ps((size_t)n * 16);
  f.read((char*)st.data(), 8 * (std::streamsize)n); f.read((char*)ps.data(), 8 * 16 * (std::streamsize)n);
  f.read((char*)&m, 4);
  std::vector<int64_t> q(m);
  f.read((char*)q.data(), 8 * (std::streamsize)m);
  if (!f) return 65;
  esvo::PoseBuffer buf;
  for (int i = 0; i < n; ++i) {
    esvo::Pose T;
    std::copy(&ps[(size_t)i * 16], &ps[(size_t)i * 16] + 16, T.begin());
    buf.setTransform(st[(size_t)i], T);
  }
  std::ofstream o(argv[2], std::ios::binary);
  for (int i = 0; i < m; ++i) {
    esvo::Pose T{};
    const int32_t found = buf.lookup(q[(size_t)i], T) ? 1 : 0;
    if (!found) T.fill(0.0);
    o.write((const char*)&found, 4); o.write((const char*)T.data(), 128);
  }
  const int32_t size = (int32_t)buf.size();
  o.write((const char*)&size, 4);
  return 0;
}
