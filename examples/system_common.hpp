// What examples/system_loop.cpp and examples/bag_system.cpp share: the hkust parameter set of the closed loop and the
// result file both write (format in system_loop.cpp's header comment).
#pragma once
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "esvo_b200/esvo_system.hpp"

namespace esvo_examples {

// esvo_time_surface/cfg/parameters.yaml + cfg/{mapping,tracking}/*_hkust.yaml (the values esvo_b200/configs.py uses)
inline esvo_params hkustParams() {
  esvo_params p; esvo_default_params(&p);
  p.decay_ms = 30.0; p.ignore_polarity = 1; p.median_blur_kernel_size = 1; p.max_event_queue_len = 20; p.time_surface_mode = 0;
  p.patch_size_x = 15; p.patch_size_y = 7; p.bm_step = 1; p.bm_zncc_threshold = 0.1; p.bm_updown = 0; p.lsnorm = ESVO_LSNORM_TDIST; p.max_iteration = 10;
  p.age_vis_threshold = 1; p.fusion_strategy = ESVO_FUSION_CONST_FRAMES; p.num_thread_mapping = 4;
  p.trk_patch_size_x = p.trk_patch_size_y = 1; p.trk_kernel_size = 5; p.trk_lsnorm = ESVO_TRK_LSNORM_HUBER; p.trk_huber_threshold = 50;
  p.trk_max_registration_points = 2000; p.trk_max_iteration = 10; p.trk_min_num_events = 1000; p.trk_batch_size = 500;
  p.invdepth_min_range = 0.25; p.invdepth_max_range = 2.0; p.residual_vis_threshold = 20; p.stdvar_vis_threshold = 0.15;
  p.fusion_radius = 0; p.max_num_fusion_frames = 20; p.max_num_fusion_points = 4000; p.smooth_time_surface = 0; p.regularization = 1;
  p.reg_radius = 5; p.reg_min_neighbours = 8; p.reg_min_close_neighbours = 8; p.td_nu = 2.1897; p.td_scale = 16.6397;
  p.bm_min_disparity = 1; p.bm_max_disparity = 40;
  return p;
}

template <class T> inline void wr(std::ofstream& o, const T* p, size_t n) { o.write((const char*)p, (std::streamsize)(n * sizeof(T))); }

// result file, trajectory, calls file (may be null) and the summary line of a finished run; 0 or the exit code
inline int writeOutputs(esvo_core::esvo_System& sys, esvo::CameraSystem& cs, bool profile, double wall_ms, const char* result,
                        const char* trajectory, const char* calls) {
  double prof_ms[8] = {0}; uint64_t prof_n[8] = {0};
  if (profile) esvo_profile_read(cs.ctx(), prof_ms, prof_n);
  std::vector<esvo::DepthPoint> map;
  sys.getMap(map);
  if (!sys.saveTrajectory(trajectory)) { std::printf("cannot write %s\n", trajectory); return 66; }

  std::ofstream o(result, std::ios::binary);
  const int32_t hdr[4] = {(int32_t)sys.ticks_.size(), (int32_t)sys.mapping_.size(), (int32_t)map.size(), sys.error_.empty() ? 0 : 1};
  wr(o, hdr, 4);
  for (const auto& tk : sys.ticks_) {
    const int32_t st[2] = {tk.status == "INITIALIZATION" ? 0 : tk.status == "WORKING" ? 1 : 2, tk.has_pose ? 1 : 0};
    const double tm[3] = {tk.ts_ms, tk.tracking_ms, tk.mapping_ms};
    wr(o, &tk.t, 1); wr(o, st, 2); wr(o, tk.T.data(), 16); wr(o, tm, 3);
  }
  for (const auto& m : sys.mapping_) {
    const int32_t a[4] = {(int32_t)m.tick, m.ran, m.ok ? 1 : 0, m.published ? 1 : 0};
    const uint64_t b[10] = {m.n_sgm_points, m.ctr.n_events, m.ctr.n_seeds, m.ctr.n_solved, m.ctr.n_culled, m.ctr.n_fusions,
                            m.ctr.bm_evals, m.ctr.lm_evals, m.ctr.map_size, m.cloud_points};
    wr(o, a, 4); wr(o, b, 10); wr(o, &m.stamp, 1);
  }
  wr(o, map.data(), map.size());
  wr(o, &wall_ms, 1); wr(o, prof_ms, 8); wr(o, prof_n, 8);
  if (calls) {
    std::FILE* cf = std::fopen(calls, "w");
    if (!cf) { std::printf("cannot write %s\n", calls); return 66; }
    for (const auto& e : sys.callTimes().ms) std::fprintf(cf, "%s %.6f %zu\n", e.first.c_str(), e.second.first, e.second.second);
    std::fclose(cf);
  }
  size_t n_pose = 0;
  for (const auto& tk : sys.ticks_) n_pose += tk.has_pose ? 1 : 0;
  std::printf("system loop: %zu ticks, %zu poses, status %s, map %zu, %.1f ms%s%s\n", sys.ticks_.size(), n_pose, sys.status_.c_str(), map.size(), wall_ms,
              sys.error_.empty() ? "" : ", stopped: ", sys.error_.c_str());
  return 0;
}

}  // namespace esvo_examples
