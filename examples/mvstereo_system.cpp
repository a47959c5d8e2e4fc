// The multi-view stereo system (include/esvo_b200/esvo_mvstereo_system.hpp) on a recorded pair of event streams with a
// stream of known poses: time surfaces and the esvo_MVStereo node in any of its five modes on one GPU, on the fixed tick
// schedule of esvo_core::esvo_MVStereoSystem.  Driven by a binary scenario so that a test can run the same stream through
// the Python restatement (tests/indep_mvstereo.py) and compare.
// usage: mvstereo_system <scenario.bin> <result.bin>
// scenario: i32 sizeof(esvo_calib), sizeof(esvo_params); esvo_calib left, right; esvo_params;
//           i64 t0_ns, dt_ns; i32 n_ticks; f64 mapping_rate_hz;
//           i32 MVStereoMode, PROCESS_EVENT_NUM, TS_HISTORY_LENGTH, EM_NUM_EVENT_MATCHING, Denoising, marker_frame, profile;
//           f64 BM_half_slice_thickness, EM_Slice_Thickness, EM_Time_THRESHOLD, EM_EPIPOLAR_THRESHOLD, EM_TS_NCC_THRESHOLD;
//           left then right events: i32 n; u16 x[n]; u16 y[n]; i64 t[n]; u8 p[n]   (time-ordered);
//           poses: i32 n; i64 stamps[n]; f64 T_world_dvs[n*16]                      (stream order)
// result:   i32 mapping frames, map size, stopped (1 = a time-surface call failed or the device reported an error after a
//           mapping pass);
//           per frame: i32 tick; i64 t; i32 gated, transferred, ran, ok, published; i64 key-frame stamp; f64 T_world_kf[16];
//                      u64 n_left, n_right, n_sgm, n_window, n_close, n_st, n_matches, cloud points, resets; f64 ms;
//           final map: esvo_depth_point[map size]; f64 wall ms; f64 stage ms[8]; u64 stage launches[8]
#include <chrono>
#include <cstdio>
#include <fstream>

#include "esvo_b200/esvo_mvstereo_system.hpp"

template <class T> static bool rd(std::ifstream& f, T* p, size_t n) { f.read((char*)p, (std::streamsize)(n * sizeof(T))); return (bool)f; }
template <class T> static void wr(std::ofstream& o, const T* p, size_t n) { o.write((const char*)p, (std::streamsize)(n * sizeof(T))); }

int main(int argc, char** argv) {
  if (argc < 3) { std::printf("usage: mvstereo_system <scenario.bin> <result.bin>\n"); return 64; }
  std::ifstream f(argv[1], std::ios::binary);
  int32_t sz[2];
  esvo_calib l{}, r{};
  esvo_params p{};
  esvo_core::esvo_MVStereoSystem::Config cfg;
  int32_t n_ticks, iv[7];
  double rate, dv[5];
  if (!rd(f, sz, 2) || sz[0] != (int32_t)sizeof(esvo_calib) || sz[1] != (int32_t)sizeof(esvo_params) || !rd(f, &l, 1) || !rd(f, &r, 1) ||
      !rd(f, &p, 1) || !rd(f, &cfg.t0_ns, 1) || !rd(f, &cfg.dt_ns, 1) || !rd(f, &n_ticks, 1) || !rd(f, &rate, 1) || !rd(f, iv, 7) ||
      !rd(f, dv, 5) || cfg.dt_ns <= 0 || rate <= 0 || iv[0] < 0 || iv[0] > 4)
    return 65;
  cfg.mapping_rate_hz = rate;
  cfg.MVStereoMode = iv[0]; cfg.PROCESS_EVENT_NUM = (size_t)iv[1]; cfg.TS_HISTORY_LENGTH = (size_t)iv[2];
  cfg.EM_NUM_EVENT_MATCHING = (size_t)iv[3]; cfg.Denoising = iv[4] != 0; cfg.marker_frame = iv[5] != 0;
  const bool profile = iv[6] != 0;
  cfg.BM_half_slice_thickness = dv[0]; cfg.EM_Slice_Thickness = dv[1]; cfg.EM_Time_THRESHOLD = dv[2];
  cfg.EM_EPIPOLAR_THRESHOLD = dv[3]; cfg.EM_TS_NCC_THRESHOLD = dv[4];
  std::vector<esvo::Event> ev[2];
  for (auto& e : ev) {
    int32_t n;
    if (!rd(f, &n, 1) || n < 0) return 65;
    std::vector<uint16_t> x(n), y(n); std::vector<int64_t> t(n); std::vector<uint8_t> pol(n);
    if (!rd(f, x.data(), n) || !rd(f, y.data(), n) || !rd(f, t.data(), n) || !rd(f, pol.data(), n)) return 65;
    e.resize(n);
    for (int i = 0; i < n; ++i) e[(size_t)i] = {x[(size_t)i], y[(size_t)i], t[(size_t)i], pol[(size_t)i] != 0};
  }
  int32_t n_pose;
  if (!rd(f, &n_pose, 1) || n_pose < 0) return 65;
  std::vector<int64_t> pt(n_pose); std::vector<double> pp((size_t)n_pose * 16);
  if (!rd(f, pt.data(), n_pose) || !rd(f, pp.data(), pp.size())) return 65;

  esvo::CameraSystem::Ptr cs;
  try { cs = std::make_shared<esvo::CameraSystem>(l, r, p, 0); }
  catch (const std::exception& e) { std::printf("%s\n", e.what()); return 2; }
  if (profile) esvo_profile(cs->ctx(), 0xff);

  esvo_core::esvo_MVStereoSystem sys(cs, cfg);
  size_t next[2] = {0, 0}, next_pose = 0;
  std::vector<esvo::Event> batch[2];
  std::vector<std::pair<int64_t, esvo::Pose>> poses;
  const auto w0 = std::chrono::steady_clock::now();
  for (int k = 0; k < n_ticks; ++k) {
    const int64_t t = sys.nextTick();
    for (int c = 0; c < 2; ++c) {   // every event with stamp < t_k not delivered yet
      batch[c].clear();
      while (next[c] < ev[c].size() && ev[c][next[c]].ts < t) batch[c].push_back(ev[c][next[c]++]);
    }
    poses.clear();
    if (sys.isMappingTick())         // every pose with stamp <= t_k not delivered yet, in stream order
      while (next_pose < pt.size() && pt[next_pose] <= t) {
        esvo::Pose T;
        std::copy(&pp[next_pose * 16], &pp[next_pose * 16] + 16, T.begin());
        poses.push_back({pt[next_pose++], T});
      }
    if (!sys.SpinOnce(batch[0], batch[1], poses)) break;
  }
  esvo_sync(cs->ctx());
  const double wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - w0).count();
  double prof_ms[8] = {0}; uint64_t prof_n[8] = {0};
  if (profile) esvo_profile_read(cs->ctx(), prof_ms, prof_n);
  std::vector<esvo::DepthPoint> map;
  sys.getMap(map);

  std::ofstream o(argv[2], std::ios::binary);
  const int32_t hdr[3] = {(int32_t)sys.frames_.size(), (int32_t)map.size(), sys.error_.empty() ? 0 : 1};
  wr(o, hdr, 3);
  size_t n_pub = 0;
  for (const auto& fr : sys.frames_) {
    const auto& q = fr.r;
    const int32_t tick = (int32_t)fr.tick;
    const int32_t b[5] = {q.gated, q.transferred, q.ran, q.ok, q.published};
    const uint64_t c[9] = {q.n_left, q.n_right, q.n_sgm, q.n_window, q.n_close, q.n_st, q.n_matches, fr.cloud_points, fr.resets};
    wr(o, &tick, 1); wr(o, &fr.t, 1); wr(o, b, 5); wr(o, &q.stamp, 1); wr(o, q.T_world_kf.data(), 16); wr(o, c, 9); wr(o, &fr.ms, 1);
    n_pub += q.published ? 1 : 0;
  }
  wr(o, map.data(), map.size());
  wr(o, &wall_ms, 1); wr(o, prof_ms, 8); wr(o, prof_n, 8);
  std::printf("mvstereo system: mode %d, %d ticks, %zu mapping frames, %zu published, map %zu, %.1f ms%s%s\n", cfg.MVStereoMode, n_ticks,
              sys.frames_.size(), n_pub, map.size(), wall_ms, sys.error_.empty() ? "" : ", stopped: ", sys.error_.c_str());
  return 0;
}
