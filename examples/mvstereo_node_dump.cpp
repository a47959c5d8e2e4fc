// What the host half of the esvo_MVStereo node (esvo_core::MVStereoFrontEnd, include/esvo_b200/esvo_core.hpp) does on a
// scripted sequence of callbacks and loop passes, for a comparison with the Python restatement (tests/indep_mvstereo.py).
// Host logic only: builds with plain g++, no library, no GPU.
// usage: mvstereo_node_dump <script.bin> <out.bin>
// script: i32 W, H, MVStereoMode, PROCESS_EVENT_NUM, TS_HISTORY_LENGTH, EM_NUM_EVENT_MATCHING, Denoising, marker_frame;
//         f64 BM_half_slice_thickness; i32 n_ops; per op i32 kind and
//           0 / 1 left / right events: i32 n; u16 x[n]; u16 y[n]; i64 t[n]; u8 p[n]
//           2 time surface: i64 stamp (the images are zeros)
//           3 pose: i64 stamp; f64 T_world_dvs[16]
//           4 one loop pass (MVStereoFrontEnd::prepare)
// out:    per op i32 kind, i32 reset (callbacks: the reset rule fired) and, for a pass:
//           i32 gated, transferred, has_obs; i64 obs stamp; f64 T_obs[16]; i64 t_low, t_up;
//           five event lists (EM left, EM right, SGM, BM window, BM denoised / truncated): i32 n; (u16 x, u16 y, i64 t)[n];
//           i32 n_st; (i64 stamp, f64 T[16])[n_st]
#include <cstdio>
#include <fstream>

#include "esvo_b200/esvo_core.hpp"

template <class T> static bool rd(std::ifstream& f, T* p, size_t n) { f.read((char*)p, (std::streamsize)(n * sizeof(T))); return (bool)f; }
template <class T> static void wr(std::ofstream& o, const T* p, size_t n) { o.write((const char*)p, (std::streamsize)(n * sizeof(T))); }

static void wrEvents(std::ofstream& o, const std::vector<esvo::Event*>& v) {
  const int32_t n = (int32_t)v.size();
  wr(o, &n, 1);
  for (const esvo::Event* e : v) { wr(o, &e->x, 1); wr(o, &e->y, 1); wr(o, &e->ts, 1); }
}

int main(int argc, char** argv) {
  if (argc < 3) { std::printf("usage: mvstereo_node_dump <script.bin> <out.bin>\n"); return 64; }
  std::ifstream f(argv[1], std::ios::binary);
  int32_t h[8], n_ops;
  double half;
  if (!rd(f, h, 8) || !rd(f, &half, 1) || !rd(f, &n_ops, 1) || h[0] <= 0 || h[1] <= 0) return 65;
  esvo_core::MVStereoFrontEnd node(h[0], h[1], h[2]);
  node.PROCESS_EVENT_NUM_ = (size_t)h[3]; node.TS_HISTORY_LENGTH_ = (size_t)h[4]; node.EM_numEventMatching_ = (size_t)h[5];
  node.bDenoising_ = h[6] != 0; node.marker_frame_ = h[7] != 0; node.BM_half_slice_thickness_ = half;
  const std::vector<uint8_t> zeros((size_t)h[0] * h[1], 0);
  std::ofstream o(argv[2], std::ios::binary);
  for (int i = 0; i < n_ops; ++i) {
    int32_t kind, reset = 0;
    if (!rd(f, &kind, 1)) return 65;
    if (kind == 0 || kind == 1) {
      int32_t n;
      if (!rd(f, &n, 1) || n < 0) return 65;
      std::vector<uint16_t> x(n), y(n); std::vector<int64_t> t(n); std::vector<uint8_t> p(n);
      if (!rd(f, x.data(), n) || !rd(f, y.data(), n) || !rd(f, t.data(), n) || !rd(f, p.data(), n)) return 65;
      std::vector<esvo::Event> ev((size_t)n);
      for (int j = 0; j < n; ++j) ev[(size_t)j] = {x[(size_t)j], y[(size_t)j], t[(size_t)j], p[(size_t)j] != 0};
      reset = node.eventsCallback(ev, kind == 0);
    } else if (kind == 2) {
      int64_t t;
      if (!rd(f, &t, 1)) return 65;
      reset = node.timeSurfaceCallback(t, zeros.data(), zeros.data());
    } else if (kind == 3) {
      int64_t t; esvo::Pose T;
      if (!rd(f, &t, 1) || !rd(f, T.data(), 16)) return 65;
      reset = node.stampedPoseCallback(t, T);
    } else if (kind != 4) {
      return 65;
    }
    wr(o, &kind, 1); wr(o, &reset, 1);
    if (kind != 4) continue;
    esvo_core::MVStereoFrontEnd::Pass p;
    node.prepare(p);
    const int32_t b[3] = {p.gated, p.transferred, p.has_obs};
    wr(o, b, 3); wr(o, &node.TS_obs_.first, 1); wr(o, node.TS_obs_.second.tr_.data(), 16);
    wr(o, &node.t_lowBound_, 1); wr(o, &node.t_upBound_, 1);
    for (const auto* v : {&node.vEventsPtr_left_, &node.vEventsPtr_right_, &node.vEventsPtr_left_SGM_, &node.vALLEventsPtr_left_,
                          &node.vDenoisedEventsPtr_left_})
      wrEvents(o, *v);
    const int32_t n_st = (int32_t)node.st_map_.size();
    wr(o, &n_st, 1);
    for (const auto& st : node.st_map_) { wr(o, &st.first, 1); wr(o, st.second.data(), 16); }
  }
  return 0;
}
