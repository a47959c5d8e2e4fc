// The closed stereo-odometry loop (include/esvo_b200/esvo_system.hpp) on a recorded pair of event streams: time surfaces,
// SGM start-up, mapping and tracking on one GPU, on the fixed tick schedule of esvo_core::esvo_System.  Driven by a binary
// scenario so that a test can run the same stream through the Python restatement (tests/indep_system.py) and compare.
// usage: system_loop <scenario.bin> <result.bin> <trajectory.txt> [calls.txt]
// scenario: i32 W, H, rig (0 hkust); i64 t0_ns, dt_ns; i32 n_ticks, mapping_every, profile (1 = per-stage esvo_profile);
//           i32 n_overrides, then (i32 key, f64 value) each -- keys: 0 trk_batch_size (BATCH_SIZE), 1 PROCESS_EVENT_NUM,
//           2 Denoising, 3 INIT_SGM_DP_NUM_THRESHOLD;
//           left then right events: i32 n; u16 x[n]; u16 y[n]; i64 t[n]; u8 p[n]   (time-ordered)
// result:   i32 ticks run, mapping records, map size, stopped (1 = a node hit a reference exit(-1));
//           per tick: i64 t; i32 status (0 INITIALIZATION, 1 WORKING, 2 TERMINATE); i32 has_pose; f64 T_world_left[16];
//                     f64 ms of events + time surfaces, of tracking, of mapping;
//           per mapping tick: i32 tick, ran (0 nothing, 1 initialisation, 2 mapping), ok, published; u64 SGM points;
//                     u64 counters[8] (esvo_mapping_at_time order); u64 published cloud points; i64 cloud stamp;
//           final map: esvo_depth_point[map size]; f64 wall ms; f64 stage ms[8]; u64 stage launches[8]
// calls:    one line per call SpinOnce / MappingLoopOnce makes: "<name> <total host ms> <calls>"
#include <chrono>
#include <cstdio>
#include <cstring>
#include <fstream>

#include "esvo_b200/esvo_system.hpp"
#include "system_common.hpp"

template <class T> static bool rd(std::ifstream& f, T* p, size_t n) { f.read((char*)p, (std::streamsize)(n * sizeof(T))); return (bool)f; }

int main(int argc, char** argv) {
  if (argc < 4) { std::printf("usage: system_loop <scenario.bin> <result.bin> <trajectory.txt> [calls.txt]\n"); return 64; }
  std::ifstream f(argv[1], std::ios::binary);
  int32_t W, H, rig, n_ticks, mapping_every, profile, n_ovr;
  int64_t t0, dt;
  if (!rd(f, &W, 1) || !rd(f, &H, 1) || !rd(f, &rig, 1) || !rd(f, &t0, 1) || !rd(f, &dt, 1) || !rd(f, &n_ticks, 1) ||
      !rd(f, &mapping_every, 1) || !rd(f, &profile, 1) || !rd(f, &n_ovr, 1) || rig != 0)
    return 65;
  // calib/hkust (the values esvo_b200/configs.py uses); parameters: cfg/{mapping,tracking}/*_hkust.yaml (system_common.hpp)
  esvo_calib l{}, r{};
  l.width = r.width = W; l.height = r.height = H;
  const double Kl[9] = {263.796, 0, 176.994, 0, 263.738, 124.373, 0, 0, 1}, Dl[4] = {-0.386589, 0.157241, 0.000322143, 6.13759e-06};
  const double Rl[9] = {0.999809, 0.0161928, 0.0109163, -0.0162088, 0.999868, 0.0013701, -0.0108927, -0.00154678, 0.999939};
  const double Pl[12] = {189.705, 0, 165.382, 0, 0, 189.705, 121.295, 0, 0, 0, 1, 0};
  const double Kr[9] = {263.485, 0, 162.942, 0, 263.276, 118.029, -0.0151344, 0.00133093, 0.999885}, Dr[4] = {-0.383425, 0.152823, -0.000257745, 0.000268432};
  const double Rr[9] = {0.9993960957463914, 0.0034732142808621717, -0.03457427641222047, -0.0035085878889783376, 0.9999933816804096,
                        -0.0009625000798637905, 0.03457070461958685, 0.0010832257094615543, 0.9994016675011942};
  double Pr[12]; std::memcpy(Pr, Pl, sizeof(Pl)); Pr[3] = -13.8634;
  std::memcpy(l.K, Kl, 72); std::memcpy(l.D, Dl, 32); std::memcpy(l.R, Rl, 72); std::memcpy(l.P, Pl, 96);
  std::memcpy(r.K, Kr, 72); std::memcpy(r.D, Dr, 32); std::memcpy(r.R, Rr, 72); std::memcpy(r.P, Pr, 96);
  esvo_params p = esvo_examples::hkustParams();
  esvo_core::esvo_System::Config cfg;
  cfg.t0_ns = t0; cfg.dt_ns = dt; cfg.mapping_every = mapping_every;
  for (int i = 0; i < n_ovr; ++i) {
    int32_t key; double v;
    if (!rd(f, &key, 1) || !rd(f, &v, 1)) return 65;
    if (key == 0) p.trk_batch_size = (int32_t)v;
    else if (key == 1) cfg.PROCESS_EVENT_NUM = (size_t)v;
    else if (key == 2) cfg.Denoising = v != 0;
    else if (key == 3) cfg.INIT_SGM_DP_NUM_THRESHOLD = (size_t)v;
    else return 65;
  }
  std::vector<esvo::Event> ev[2];
  for (auto& e : ev) {
    int32_t n;
    if (!rd(f, &n, 1)) return 65;
    std::vector<uint16_t> x(n), y(n); std::vector<int64_t> t(n); std::vector<uint8_t> pol(n);
    if (!rd(f, x.data(), n) || !rd(f, y.data(), n) || !rd(f, t.data(), n) || !rd(f, pol.data(), n)) return 65;
    e.resize(n);
    for (int i = 0; i < n; ++i) e[(size_t)i] = {x[(size_t)i], y[(size_t)i], t[(size_t)i], pol[(size_t)i] != 0};
  }
  esvo::CameraSystem::Ptr cs;
  try { cs = std::make_shared<esvo::CameraSystem>(l, r, p, 0); }
  catch (const std::exception& e) { std::printf("%s\n", e.what()); return 2; }
  if (profile) esvo_profile(cs->ctx(), 0xff);

  esvo_core::esvo_System sys(cs, cfg);
  size_t next[2] = {0, 0};
  std::vector<esvo::Event> batch[2];
  const auto w0 = std::chrono::steady_clock::now();
  for (int k = 0; k < n_ticks; ++k) {
    const int64_t t = sys.nextTick();
    for (int c = 0; c < 2; ++c) {   // every event with stamp < t_k not delivered yet
      batch[c].clear();
      while (next[c] < ev[c].size() && ev[c][next[c]].ts < t) batch[c].push_back(ev[c][next[c]++]);
    }
    if (!sys.SpinOnce(batch[0], batch[1])) break;
  }
  esvo_sync(cs->ctx());
  const double wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - w0).count();
  return esvo_examples::writeOutputs(sys, *cs, profile != 0, wall_ms, argv[2], argv[3], argc > 4 ? argv[4] : nullptr);
}
