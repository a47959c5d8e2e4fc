// esvo_b200 product code -- C ABI, part 2: culling, fusion, map and whole-frame mapping entry points.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "common.cuh"
#include "sgbm_core.h"

namespace esvo {
int fuse_zero_fusion_counter(Ctx* c);
int fuse_fetch_scalars(Ctx* c, unsigned long long out[4]);
int fuse_reserve(Ctx* c, size_t total_points);
int fuse_window(Ctx* c, const Ctx::WinFrame* frames, int nframes, int radius);
int sgbm_run(Ctx* c, const uint8_t* d_left, const uint8_t* d_right, int pitch, const esvo_sgbm::Dims& dm, int16_t* d_out);

// Window vectors are recycled through a FIFO pool.  A vector popped from the window may still be read by the
// fusion of the frame that preceded the pop (running on another slot's stream), so it carries an event recorded
// behind that fusion, and it is only reused after `depth` further frames: the wait below is then already satisfied.
static int win_acquire(Ctx* c, size_t cap, Ctx::WinFrame& f) {
  if (c->win_pool.size() > (size_t)c->depth)
    for (size_t i = 0; i < c->win_pool.size() - (size_t)c->depth; ++i)
      if (c->win_pool[i].cap >= cap) {
        f = c->win_pool[i]; c->win_pool.erase(c->win_pool.begin() + i);
        if (f.last_read) ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->stream, f.last_read, 0));
        return ESVO_OK;
      }
  f = Ctx::WinFrame();
  f.cap = std::max<size_t>(cap, 1024);
  ESVO_CUDA_TRY(c, dmalloc(&f.pts, f.cap));
  ESVO_CUDA_TRY(c, dmalloc(&f.cnt, 1));
  ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&f.last_read, cudaEventDisableTiming));
  return ESVO_OK;
}
static int win_retire(Ctx* c, Ctx::WinFrame f) {
  // last reader = the fusion of the previous frame (frame_no - 1), enqueued on that frame's slot stream
  if (c->frame_no >= 1 && f.last_read) {
    cudaStream_t st = c->slots[(int)((c->frame_no - 1) % (uint64_t)c->depth)].stream;
    if (st) ESVO_CUDA_TRY(c, cudaEventRecord(f.last_read, st));
  }
  c->win_pool.push_back(f);
  return ESVO_OK;
}

// esvo_Mapping::MappingAtTime (esvo_Mapping.cpp:261-399), kernels only, everything stays on the device.
static int run_mapping_frame(Ctx* c) {
  const esvo_params& p = c->prm;
  int rc;
  SlotBufs& sl = c->slot();
  ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->stream, sl.ev_obs, 0));        // observation of this frame is in place
  cudaEvent_t pe = c->prof_begin(1);
  if (p.smooth_time_surface && (rc = smooth_obs(c))) return rc;           // createMatchProblem (EventBM.cpp:68-72)
  ESVO_CUDA_TRY(c, cudaMemsetAsync(sl.d_counters, 0, kCounters * 8, c->stream));
  if ((rc = bm_run(c))) return rc;                                        // :308-309
  c->prof_end(pe); pe = c->prof_begin(2);
  if ((rc = seeds_order(c))) return rc;
  c->prof_end(pe);
  // (Giving the LM kernel its own low-priority stream and the short stages high-priority streams made the pipeline
  //  slower and erratic when it was tried, so everything of a frame stays on the slot's single stream.)
  pe = c->prof_begin(3);
  if ((rc = lm_run(c, sl.d_seeds, 0))) return rc;                         // :330
  c->prof_end(pe);
  ESVO_CUDA_TRY(c, cudaEventRecord(sl.ev_free, c->stream));               // the slot's observation buffers are free again
  sl.ev_free_valid = true;
  Ctx::WinFrame f;
  if ((rc = win_acquire(c, std::max<size_t>(sl.n_ev, 1), f))) return rc;
  const double cost_thr = p.residual_vis_threshold * p.residual_vis_threshold * (double)(p.patch_size_x * p.patch_size_y);
  pe = c->prof_begin(4);
  if ((rc = points_order_impl(c, sl.d_seeds, 0, 1, p.stdvar_vis_threshold, cost_thr, p.invdepth_min_range,
                              p.invdepth_max_range, f.pts, f.cnt)))       // :334 pointCulling
    return rc;
  c->prof_end(pe);
  c->win.push_back(f);                                                    // :342-368
  if (p.fusion_strategy == ESVO_FUSION_CONST_POINTS) {
    // needs the per-frame counts on the host: one small D2H per frame (the reference's CONST_FRAMES cfgs avoid it)
    auto total = [&](size_t& tot) -> int {
      tot = 0;
      for (auto& w : c->win) {
        unsigned long long n = 0;
        ESVO_CUDA_TRY(c, cudaMemcpyAsync(&n, w.cnt, 8, cudaMemcpyDeviceToHost, c->stream));
        ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        tot += (size_t)n;
      }
      return ESVO_OK;
    };
    size_t tot;
    if ((rc = total(tot))) return rc;
    while ((double)tot > 1.5 * p.max_num_fusion_points && !c->win.empty()) {
      if ((rc = win_retire(c, c->win.front()))) return rc;
      c->win.erase(c->win.begin());
      if ((rc = total(tot))) return rc;
    }
  } else {
    while (c->win.size() > (size_t)p.max_num_fusion_frames) {
      if ((rc = win_retire(c, c->win.front()))) return rc;
      c->win.erase(c->win.begin());
    }
  }
  // The window holds vectors written by the point-ordering kernels of the previous frames, which run on other slots'
  // streams and may finish later than ours (LM tails).  Chain the "points ready" events: ev_pts of frame k is recorded
  // behind a wait on ev_pts of frame k-1, so waiting on one event covers every older vector (one wait instead of depth-1).
  if (c->depth > 1 && c->frame_no >= 1) {
    SlotBufs& prev = c->slots[(int)((c->frame_no - 1) % (uint64_t)c->depth)];
    if (prev.ev_pts_valid) ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->stream, prev.ev_pts, 0));
  }
  ESVO_CUDA_TRY(c, cudaEventRecord(sl.ev_pts, c->stream));
  sl.ev_pts_valid = true;
  pe = c->prof_begin(5);
  if ((rc = fuse_reset_map(c, sl.T_world_left))) return rc;               // :268-272 fresh DepthFrame at the obs pose
  {  // size the staging area once for a full window so that steady-state frames never reallocate
    size_t tot = 0, mx = 0;
    for (auto& w : c->win) { tot += w.cap; mx = std::max(mx, w.cap); }
    if (p.fusion_strategy == ESVO_FUSION_CONST_FRAMES) tot = std::max(tot, mx * (size_t)std::max(1, p.max_num_fusion_frames));
    if ((rc = fuse_reserve(c, tot))) return rc;
  }
  {                                                                       // :372-377 newest first
    Ctx::WinFrame order[64];
    std::vector<Ctx::WinFrame> big;
    const Ctx::WinFrame* ord = order;
    const size_t nw = c->win.size();
    if (nw <= 64) for (size_t i = 0; i < nw; ++i) order[i] = c->win[nw - 1 - i];
    else { big.assign(c->win.rbegin(), c->win.rend()); ord = big.data(); }
    if ((rc = fuse_window(c, ord, (int)nw, p.fusion_radius))) return rc;
  }
  {
    // :385-386 SmartGrid::clean once the window is full -- applied by the fold itself to the pixels it finishes
    const double clean4[4] = {p.stdvar_vis_threshold * p.stdvar_vis_threshold, p.age_vis_threshold, p.invdepth_max_range, p.invdepth_min_range};
    const bool do_clean = c->win.size() >= (size_t)p.max_num_fusion_frames;
    if ((rc = fuse_finish(c, false, do_clean ? clean4 : nullptr))) return rc;
  }
  if (p.regularization) rc = map_regularize(c, /*count=*/true);           // :390-395, + element count
  else rc = map_count(c);
  c->prof_end(pe);
  ESVO_CUDA_TRY(c, cudaEventRecord(sl.ev_fuse, c->stream));
  sl.ev_fuse_valid = true;
  c->frame_no++;
  return rc;
}

// The 8-counter record of a mapping frame {n_events, n_seeds, n_solved, n_culled, n_fusions, bm_evals, lm_evals, map_size}
// from the slot's fetched counters and its map scalars (fuse_fetch_scalars: [0] = n_fusions, [2] = map size).
static void mapping_counters(const SlotBufs& s, const unsigned long long map_scal[4], uint64_t out[8]) {
  out[0] = s.n_ev; out[1] = s.h_counters[1]; out[2] = s.h_counters[2]; out[3] = s.h_counters[3];
  out[4] = map_scal[0]; out[5] = s.h_counters[5]; out[6] = s.h_counters[6]; out[7] = map_scal[2];
}
static int fetch_mapping_counters(Ctx* c, uint64_t out[8]) {
  int rc = fetch_counters(c);
  if (rc) return rc;
  unsigned long long sc[4];
  if ((rc = fuse_fetch_scalars(c, sc))) return rc;
  mapping_counters(c->slot(), sc, out);
  return ESVO_OK;
}
// The slot holding results_begin's ticket, once its hand-off has landed.  Slots need not rotate (the host esvo_set_ts_pair
// keeps one), so every slot is searched.
static int ticket_slot(Ctx* c, int64_t ticket, const char* who, SlotBufs** out) {
  for (SlotBufs& s : c->slots)
    if (s.dl_ticket == ticket) {
      ESVO_CUDA_TRY(c, cudaEventSynchronize(s.ev_dl));
      *out = &s;
      return ESVO_OK;
    }
  c->set_error(std::string(who) + ": unknown ticket");
  return ESVO_ERR_STATE;
}
}  // namespace esvo

using namespace esvo;

extern "C" {

ESVO_API int esvo_depth_cull(esvo_ctx* c, esvo_depth_point* pts, size_t* n, double std_thr, double cost_thr,
                             double rmin, double rmax) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  if (!n || (*n && !pts)) return ESVO_ERR_INVALID_ARG;
  if (*n == 0) return ESVO_OK;
  SlotBufs& f = c->slot();
  int rc = map_alloc_inputs(c, std::max(*n, f.n_ev), f.n_poses);
  if (rc) return rc;
  esvo_depth_point* tmp = nullptr;
  ESVO_CUDA_TRY(c, dmalloc(&tmp, *n));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(tmp, pts, *n * sizeof(esvo_depth_point), cudaMemcpyHostToDevice, c->stream));
  rc = cull_points(c, tmp, *n, std_thr, cost_thr, rmin, rmax);
  if (!rc) rc = fetch_counters(c);
  if (!rc) {
    const size_t cnt = (size_t)f.h_counters[3];
    if (cnt) cudaMemcpy(pts, f.d_pts, cnt * sizeof(esvo_depth_point), cudaMemcpyDeviceToHost);
    *n = cnt;
  }
  cudaFree(tmp);
  return rc;
}

ESVO_API int esvo_fuse(esvo_ctx* c, const esvo_depth_point* pts, size_t n, const double T[16], int radius, int reset_map,
                       int* n_fusions) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  if (n && !pts) return ESVO_ERR_INVALID_ARG;
  int rc;
  if (reset_map) { if (!T) return ESVO_ERR_INVALID_ARG; if ((rc = fuse_reset_map(c, T))) return rc; }
  if ((rc = fuse_zero_fusion_counter(c))) return rc;
  esvo_depth_point* tmp = nullptr;
  if (n) {
    ESVO_CUDA_TRY(c, dmalloc(&tmp, n));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(tmp, pts, n * sizeof(esvo_depth_point), cudaMemcpyHostToDevice, c->stream));
    rc = fuse_points(c, tmp, n, nullptr, radius, 0);
    if (!rc) rc = fuse_finish(c);
  }
  unsigned long long sc[4] = {0, 0, 0, 0};
  if (!rc) rc = fuse_fetch_scalars(c, sc);
  if (tmp) cudaFree(tmp);
  if (n_fusions) *n_fusions = (int)sc[0];
  return rc;
}

// ---- comparison modes of esvo_MVStereo (SURVEY 8f row 4) ----
ESVO_API int esvo_em_match(esvo_ctx* c, const esvo_em_params* prm, const uint16_t* lx, const uint16_t* ly, const int64_t* lt, const uint8_t* lp,
                           size_t nl, const int32_t* slice_counts, const double* slice_poses, size_t n_slices, const uint16_t* rx,
                           const uint16_t* ry, const int64_t* rt, const uint8_t* rp, size_t nr, esvo_seed* out, size_t* n_seeds,
                           uint64_t* n_evals) {
  CHECK_CTX(c);
  if (!prm || !n_seeds || (nl && (!lx || !ly || !lt || !lp)) || (nr && (!rx || !ry || !rt || !rp)) || (n_slices && (!slice_counts || !slice_poses)))
    return ESVO_ERR_INVALID_ARG;
  if (prm->patch_size_x < 1 || prm->patch_size_y < 1 || (*n_seeds && !out)) return ESVO_ERR_INVALID_ARG;
  { int rc0 = drain(c); if (rc0) return rc0; }
  if (!c->obs_set) return ESVO_ERR_STATE;
  return em_match(c, prm, lx, ly, lt, lp, nl, slice_counts, slice_poses, n_slices, rx, ry, rt, rp, nr, out, n_seeds, n_evals);
}
ESVO_API int esvo_seeds_to_points(esvo_ctx* c, const esvo_seed* seeds, size_t n, esvo_depth_point* out) {
  CHECK_CTX(c);
  if (n && (!seeds || !out)) return ESVO_ERR_INVALID_ARG;
  { int rc0 = drain(c); if (rc0) return rc0; }
  return seeds_to_points(c, seeds, n, out);
}
ESVO_API int esvo_naive_propagate(esvo_ctx* c, const esvo_depth_point* pts, size_t n, const double T[16], int reset_map) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  if (n && !pts) return ESVO_ERR_INVALID_ARG;
  int rc = ESVO_OK;
  if (reset_map) { if (!T) return ESVO_ERR_INVALID_ARG; if ((rc = fuse_reset_map(c, T))) return rc; }
  esvo_depth_point* tmp = nullptr;
  if (n) {
    ESVO_CUDA_TRY(c, dmalloc(&tmp, n));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(tmp, pts, n * sizeof(esvo_depth_point), cudaMemcpyHostToDevice, c->stream));
    rc = fuse_points(c, tmp, n, nullptr, 0, /*naive=*/1);
    if (!rc) rc = fuse_finish(c, /*naive=*/true);
    cudaError_t e = cudaStreamSynchronize(c->stream);
    cudaFree(tmp);
    if (!rc && e != cudaSuccess) { c->set_error(std::string("esvo_naive_propagate: ") + cudaGetErrorString(e)); rc = ESVO_ERR_CUDA; }
  }
  return rc;
}

ESVO_API int esvo_map_clean(esvo_ctx* c, double var_thr, double age_thr, double rmax, double rmin) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  return map_clean(c, var_thr, age_thr, rmax, rmin);
}
ESVO_API int esvo_map_regularize(esvo_ctx* c) { CHECK_CTX(c); if (int rc0 = drain_if_pipelined(c)) return rc0; return map_regularize(c); }
ESVO_API int esvo_map_download(esvo_ctx* c, esvo_depth_point* out, size_t* n) {
  CHECK_CTX(c);
  if (!n) return ESVO_ERR_INVALID_ARG;
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  return map_download(c, out, n);
}
ESVO_API int esvo_map_publish_dev(esvo_ctx* c, const double T[16], int64_t stamp, size_t* n_points) {
  CHECK_CTX(c);
  if (!T || !n_points) return ESVO_ERR_INVALID_ARG;
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  c->pub.valid = false;
  int rc = map_publish(c, T, n_points);
  if (rc) return rc;
  c->pub.n = *n_points; c->pub.stamp = stamp; c->pub.valid = true;
  return ESVO_OK;
}
ESVO_API int esvo_map_published_cloud_dev(esvo_ctx* c, float* xyz_dev, size_t* n, int64_t* stamp) {
  CHECK_CTX(c);
  if (!n) return ESVO_ERR_INVALID_ARG;
  if (!c->pub.valid) { c->set_error("esvo_map_published_cloud_dev: no cloud was published on this context"); return ESVO_ERR_STATE; }
  if (c->pub.n > *n) { *n = c->pub.n; return ESVO_ERR_CAPACITY; }
  if (c->pub.n && !xyz_dev) return ESVO_ERR_INVALID_ARG;
  if (c->pub.n) ESVO_CUDA_TRY(c, cudaMemcpyAsync(xyz_dev, c->pub.xyz, c->pub.n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  *n = c->pub.n;
  if (stamp) *stamp = c->pub.stamp;
  return ESVO_OK;
}
ESVO_API int esvo_sgbm_compute(esvo_ctx* c, const uint8_t* left, const uint8_t* right, int num_disparities, int block_size, int P1, int P2,
                               int disp12_max_diff, int pre_filter_cap, int uniqueness_ratio, int16_t* disp16_out) {
  CHECK_CTX(c);
  if (!disp16_out || (left == nullptr) != (right == nullptr)) return ESVO_ERR_INVALID_ARG;
  const int W = c->dc.W, H = c->dc.H;
  if (num_disparities <= 0 || num_disparities > esvo_sgbm::kMaxD || num_disparities >= W) {
    c->set_error("esvo_sgbm_compute: numDisparities must be in [1, 128] and smaller than the image width");
    return ESVO_ERR_UNSUPPORTED;
  }
  { int rc0 = drain(c); if (rc0) return rc0; }                     // a one-off at start-up: strictly synchronous
  const esvo_sgbm::Dims dm = esvo_sgbm::make_dims(W, H, num_disparities, block_size, P1, P2, disp12_max_diff, pre_filter_cap, uniqueness_ratio);
  uint8_t *d_l = nullptr, *d_r = nullptr; int16_t* d_out = nullptr;
  const uint8_t *src_l, *src_r; int pitch;
  auto cleanup = [&]() { cudaFree(d_l); cudaFree(d_r); cudaFree(d_out); };
  if (dmalloc(&d_out, (size_t)W * H)) { cleanup(); return ESVO_ERR_CUDA; }
  if (left) {
    if (dmalloc(&d_l, (size_t)W * H) || dmalloc(&d_r, (size_t)W * H)) { cleanup(); return ESVO_ERR_CUDA; }
    cudaError_t ce = cudaMemcpyAsync(d_l, left, (size_t)W * H, cudaMemcpyHostToDevice, c->stream);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_r, right, (size_t)W * H, cudaMemcpyHostToDevice, c->stream);
    if (ce != cudaSuccess) { cleanup(); c->set_error(cudaGetErrorString(ce)); return ESVO_ERR_CUDA; }
    src_l = d_l; src_r = d_r; pitch = W;
  } else {                                                         // the observation pair that is already on the device
    if (!c->obs_set) { cleanup(); return ESVO_ERR_STATE; }
    src_l = c->slot().obs_l; src_r = c->slot().obs_r; pitch = c->dc.pitch;
  }
  int rc = sgbm_run(c, src_l, src_r, pitch, dm, d_out);
  if (rc == ESVO_OK && cudaMemcpy(disp16_out, d_out, (size_t)W * H * 2, cudaMemcpyDeviceToHost) != cudaSuccess) rc = ESVO_ERR_CUDA;
  cleanup();
  return rc;
}

}  // extern "C"

// InitializationAtTime downstream of the SGM (esvo_Mapping.cpp:433-492) on events that are on the device already (ex_dev / ey_dev),
// or, with ex / ey, on host events uploaded first.
static int init_from_disparity(esvo_ctx* c, const int16_t* disp16, const uint16_t* ex, const uint16_t* ey, const uint16_t* ex_dev,
                               const uint16_t* ey_dev, size_t n, const double T[16], size_t min_points, size_t* n_points, int* accepted) {
  { int rc0 = drain(c); if (rc0) return rc0; }                     // a one-off at start-up: strictly synchronous
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  int16_t* d_disp = nullptr; uint16_t *d_x = nullptr, *d_y = nullptr;
  Ctx::WinFrame f;
  int rc = win_acquire(c, std::max<size_t>(n, 1), f);
  if (rc) return rc;
  auto cleanup = [&]() { cudaFree(d_disp); cudaFree(d_x); cudaFree(d_y); };
  if (dmalloc(&d_disp, npix) || (!ex_dev && (dmalloc(&d_x, n) || dmalloc(&d_y, n)))) { cleanup(); c->win_pool.push_back(f); return ESVO_ERR_CUDA; }
  cudaError_t ce = cudaMemcpyAsync(d_disp, disp16, npix * 2, cudaMemcpyHostToDevice, c->stream);
  if (!ex_dev && n && ce == cudaSuccess) ce = cudaMemcpyAsync(d_x, ex, n * 2, cudaMemcpyHostToDevice, c->stream);
  if (!ex_dev && n && ce == cudaSuccess) ce = cudaMemcpyAsync(d_y, ey, n * 2, cudaMemcpyHostToDevice, c->stream);
  if (ce != cudaSuccess) { cleanup(); c->win_pool.push_back(f); c->set_error(cudaGetErrorString(ce)); return ESVO_ERR_CUDA; }
  unsigned long long cnt = 0;
  const uint16_t* px = ex_dev ? ex_dev : d_x;
  const uint16_t* py = ex_dev ? ey_dev : d_y;
  if ((rc = fuse_reset_map(c, T)) == ESVO_OK && (rc = sgm_points(c, d_disp, px, py, n, f.pts, f.cnt)) == ESVO_OK) {
    if (cudaMemcpyAsync(&cnt, f.cnt, 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess)
      rc = ESVO_ERR_CUDA;
  }
  cleanup();
  if (rc) { c->win_pool.push_back(f); return rc; }
  if (n_points) *n_points = (size_t)cnt;
  if (cnt < min_points) {                                          // esvo_Mapping.cpp:481-483
    c->win_pool.push_back(f);
    if (accepted) *accepted = 0;
    return ESVO_OK;
  }
  c->win.push_back(f);                                             // :485 dqvDepthPoints_.push_back(vdp_sgm)
  std::memcpy(c->slot().T_world_left, T, sizeof(SlotBufs::T_world_left));
  if ((rc = fuse_zero_fusion_counter(c))) return rc;
  if ((rc = fuse_points(c, f.pts, (size_t)cnt, nullptr, 0, /*naive=*/1))) return rc;   // :486 naive_propagation
  if ((rc = fuse_finish(c, true))) return rc;
  if ((rc = map_count(c))) return rc;
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (accepted) *accepted = 1;
  return ESVO_OK;
}

extern "C" {

ESVO_API int esvo_init_from_disparity(esvo_ctx* c, const int16_t* disp16, const uint16_t* ex, const uint16_t* ey, size_t n,
                                      const double T[16], size_t min_points, size_t* n_points, int* accepted) {
  CHECK_CTX(c);
  if (!disp16 || !T || (n && (!ex || !ey))) return ESVO_ERR_INVALID_ARG;
  return init_from_disparity(c, disp16, ex, ey, nullptr, nullptr, n, T, min_points, n_points, accepted);
}

// ---- event windows read from the time-surface log (events.cu) ----
ESVO_API int esvo_events_window_dev(esvo_ctx* c, int cam, int64_t front, int64_t t_begin_ns, int64_t t_end_ns, size_t budget, int denoise,
                                    size_t max_keep, size_t* n) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  return events_window(c, cam, front, t_begin_ns, t_end_ns, budget, denoise, max_keep, n);
}
ESVO_API int esvo_events_lower_bound_dev(esvo_ctx* c, int cam, int64_t front, const int64_t* t_ns, size_t k, int64_t* idx_out) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || (k && (!t_ns || !idx_out))) return ESVO_ERR_INVALID_ARG;
  return events_lower_bound(c, cam, front, t_ns, k, idx_out);
}
ESVO_API int esvo_events_selected_dev(esvo_ctx* c, uint16_t* x_dev, uint16_t* y_dev, int64_t* t_dev, size_t* n) {
  CHECK_CTX(c);
  if (!n) return ESVO_ERR_INVALID_ARG;
  const Ctx::EventWindow& w = c->evw;
  if (!w.valid) { c->set_error("esvo_events_selected_dev: no event window was selected on this context"); return ESVO_ERR_STATE; }
  if (w.n > *n) { *n = w.n; return ESVO_ERR_CAPACITY; }
  if (w.n && (!x_dev || !y_dev || !t_dev)) return ESVO_ERR_INVALID_ARG;
  if (w.n) {
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(x_dev, w.kx, w.n * 2, cudaMemcpyDeviceToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(y_dev, w.ky, w.n * 2, cudaMemcpyDeviceToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(t_dev, w.kt, w.n * 8, cudaMemcpyDeviceToDevice, c->stream));
  }
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  *n = w.n;
  return ESVO_OK;
}
ESVO_API int esvo_mapping_at_time_selected_dev(esvo_ctx* c, const int64_t* pt, const double* poses, size_t np, uint64_t* counters) {
  CHECK_CTX(c);
  if (np && (!pt || !poses)) return ESVO_ERR_INVALID_ARG;
  if (c->depth > 1) { c->set_error("esvo_mapping_at_time_selected_dev: not available at pipeline depth > 1"); return ESVO_ERR_STATE; }
  const Ctx::EventWindow& w = c->evw;
  if (!w.valid) { c->set_error("esvo_mapping_at_time_selected_dev: no event window was selected on this context"); return ESVO_ERR_STATE; }
  if (!c->obs_set) return ESVO_ERR_STATE;
  int rc = map_alloc_inputs(c, w.n, np);
  if (rc) return rc;
  if ((rc = stage_inputs_packed(c, nullptr, nullptr, nullptr, 0, pt, poses, np))) return rc;   // the poses only
  SlotBufs& f = c->slot();
  f.n_ev = w.n; f.d_ex = w.kx; f.d_ey = w.ky; f.d_et = w.kt;                                      // the events in place
  if ((rc = esvo_run_mapping(c))) return rc;
  uint64_t ctr[8];
  if ((rc = fetch_mapping_counters(c, ctr))) return rc;
  if (counters) std::memcpy(counters, ctr, sizeof(ctr));
  return ESVO_OK;
}
ESVO_API int esvo_init_from_disparity_selected_dev(esvo_ctx* c, const int16_t* disp16, const double T[16], size_t min_points, size_t* n_points,
                                                   int* accepted) {
  CHECK_CTX(c);
  if (!disp16 || !T) return ESVO_ERR_INVALID_ARG;
  if (c->depth > 1) { c->set_error("esvo_init_from_disparity_selected_dev: not available at pipeline depth > 1"); return ESVO_ERR_STATE; }
  const Ctx::EventWindow& w = c->evw;
  if (!w.valid) { c->set_error("esvo_init_from_disparity_selected_dev: no event window was selected on this context"); return ESVO_ERR_STATE; }
  return init_from_disparity(c, disp16, nullptr, nullptr, w.kx, w.ky, w.n, T, min_points, n_points, accepted);
}

ESVO_API int esvo_window_download(esvo_ctx* c, int index, esvo_depth_point* out, size_t* n) {
  CHECK_CTX(c);
  if (!n || index < 0) return ESVO_ERR_INVALID_ARG;
  { int rc0 = drain(c); if (rc0) return rc0; }
  if ((size_t)index >= c->win.size()) { *n = 0; return ESVO_ERR_INVALID_ARG; }
  const Ctx::WinFrame& f = c->win[(size_t)index];
  unsigned long long cnt = 0;
  ESVO_CUDA_TRY(c, cudaMemcpy(&cnt, f.cnt, 8, cudaMemcpyDeviceToHost));
  if (cnt > *n) { *n = (size_t)cnt; return ESVO_ERR_CAPACITY; }
  if (cnt && !out) return ESVO_ERR_INVALID_ARG;
  if (cnt) ESVO_CUDA_TRY(c, cudaMemcpy(out, f.pts, (size_t)cnt * sizeof(esvo_depth_point), cudaMemcpyDeviceToHost));
  *n = (size_t)cnt;
  return ESVO_OK;
}

ESVO_API int esvo_mapping_reset(esvo_ctx* c) {
  CHECK_CTX(c);
  { int rc0 = drain(c); if (rc0) return rc0; }
  for (auto& f : c->win) c->win_pool.push_back(f);   // drained above: no reader is pending
  c->win.clear();
  return ESVO_OK;
}

ESVO_API int esvo_stage_mapping_inputs(esvo_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et, size_t n,
                                       const int64_t* pt, const double* poses, size_t np) {
  CHECK_CTX(c);
  if (n && (!ex || !ey || !et)) return ESVO_ERR_INVALID_ARG;
  if (np && (!pt || !poses)) return ESVO_ERR_INVALID_ARG;
  return stage_inputs_packed(c, ex, ey, et, n, pt, poses, np);    // the caller's arrays are free again on return
}
// Device-resident inputs are used IN PLACE (no copy): they must stay valid and unchanged until the frame has been
// collected (esvo_results_end) or the ctx synchronised.
ESVO_API int esvo_stage_mapping_inputs_dev(esvo_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et, size_t n,
                                           const int64_t* pt, const double* poses, size_t np) {
  CHECK_CTX(c);
  if (n && (!ex || !ey || !et)) return ESVO_ERR_INVALID_ARG;
  if (np && (!pt || !poses)) return ESVO_ERR_INVALID_ARG;
  int rc = map_alloc_inputs(c, n, np);
  if (rc) return rc;
  SlotBufs& f = c->slot();
  f.n_ev = n; f.n_poses = np;
  f.d_ex = const_cast<uint16_t*>(ex); f.d_ey = const_cast<uint16_t*>(ey); f.d_et = const_cast<int64_t*>(et);
  f.d_pose_t = const_cast<int64_t*>(pt); f.d_poses = const_cast<double*>(poses);
  return ESVO_OK;
}
// ---- asynchronous result hand-off for pipelined operation ----
ESVO_API int esvo_results_begin(esvo_ctx* c, int64_t* ticket_out) {
  CHECK_CTX(c);
  if (c->frame_no == 0) return ESVO_ERR_STATE;
  SlotBufs& sl = c->slot();
  if (sl.dl_ticket >= 0) { c->set_error("esvo_results_begin: the previous results of this pipeline slot were not collected"); return ESVO_ERR_STATE; }
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  if (!sl.d_dl) {
    // first use: set up the result buffers of EVERY pipeline slot now (pinned allocations take milliseconds each
    // and must not land in the middle of a running pipeline)
    for (int i = 0; i < c->depth; ++i) {
      SlotBufs& q = c->slots[i];
      if (q.d_dl) continue;
      ESVO_CUDA_TRY(c, dmalloc(&q.d_dl, npix)); ESVO_CUDA_TRY(c, dmalloc(&q.d_dl_keys, npix)); ESVO_CUDA_TRY(c, dmalloc(&q.d_dlscal, 4));
      ESVO_CUDA_TRY(c, cudaMallocHost((void**)&q.h_dlscal, 8 * 8));
      ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&q.ev_dl, cudaEventDisableTiming));
      // ordered results land here straight from the gather kernels (pinned memory is device-accessible under UVA)
      q.h_dl_bytes = npix * sizeof(esvo_depth_point);
      ESVO_CUDA_TRY(c, cudaHostAlloc(&q.h_dl, q.h_dl_bytes, cudaHostAllocDefault));
    }
  }
  if (!c->s_copy) ESVO_CUDA_TRY(c, cudaStreamCreateWithFlags(&c->s_copy, cudaStreamNonBlocking));
  {
    // right behind this frame's fusion on the slot's own stream
    int rc = map_gather_async(c, sl.d_dl, sl.d_dl_keys, sl.d_dlscal, sl.h_dlscal, (esvo_depth_point*)sl.h_dl, sl.h_counters);
    if (rc) return rc;
    ESVO_CUDA_TRY(c, cudaEventRecord(sl.ev_dl, c->stream));
  }
  sl.dl_ticket = (int64_t)c->frame_no - 1;
  if (ticket_out) *ticket_out = sl.dl_ticket;
  return ESVO_OK;
}
ESVO_API int esvo_results_end(esvo_ctx* c, int64_t ticket, esvo_depth_point* out, size_t* n, uint64_t counters[8]) {
  CHECK_CTX(c);
  if (!n || ticket < 0) return ESVO_ERR_INVALID_ARG;
  SlotBufs* sl;
  if (int rc = ticket_slot(c, ticket, "esvo_results_end", &sl)) return rc;
  const size_t cnt = (size_t)sl->h_dlscal[1];
  if (counters) mapping_counters(*sl, sl->h_dlscal + 4, counters);
  if (cnt > *n) { *n = cnt; return ESVO_ERR_CAPACITY; }
  if (cnt && !out) return ESVO_ERR_INVALID_ARG;
  std::memcpy(out, sl->h_dl, cnt * sizeof(esvo_depth_point));   // already in SmartGrid list order (creation sequence)
  *n = cnt;
  sl->dl_ticket = -1;
  return ESVO_OK;
}
// Zero-copy form: *out points into the slot's pinned landing buffer (written by the gather kernel over PCIe); valid until the
// slot issues its next esvo_results_begin.
ESVO_API int esvo_results_end_view(esvo_ctx* c, int64_t ticket, const esvo_depth_point** out, size_t* n, uint64_t counters[8]) {
  CHECK_CTX(c);
  if (!n || !out || ticket < 0) return ESVO_ERR_INVALID_ARG;
  SlotBufs* sl;
  if (int rc = ticket_slot(c, ticket, "esvo_results_end_view", &sl)) return rc;
  if (counters) mapping_counters(*sl, sl->h_dlscal + 4, counters);
  *out = (const esvo_depth_point*)sl->h_dl;
  *n = (size_t)sl->h_dlscal[1];
  sl->dl_ticket = -1;
  return ESVO_OK;
}
ESVO_API uint64_t esvo_debug_counter(esvo_ctx* c, int idx) { return (c && idx >= 0 && idx < kCounters) ? c->slot().h_counters[idx] : 0; }
ESVO_API int esvo_profile(esvo_ctx* c, int stage_mask) {
  CHECK_CTX(c);
  c->prof = (unsigned)stage_mask & 0xffu;
  // Events are created here, not on the hot path: enough for ~512 records before the next esvo_profile_read.
  if (c->prof) while (c->prof_pool.size() < 1024) { cudaEvent_t e; ESVO_CUDA_TRY(c, cudaEventCreate(&e)); c->prof_pool.push_back(e); }
  return ESVO_OK;
}
// Debug: dump every recorded (stage, begin, end) as a timeline in ms relative to the earliest event.
ESVO_API int esvo_profile_dump(esvo_ctx* c, const char* path) {
  CHECK_CTX(c);
  int rc0 = drain(c);
  if (rc0) return rc0;
  cudaEvent_t ref = nullptr;
  for (int s = 0; s < 8 && !ref; ++s) if (!c->prof_ev[s].empty()) ref = c->prof_ev[s][0].first;
  if (!ref) return ESVO_ERR_STATE;
  FILE* f = fopen(path, "w");
  if (!f) return ESVO_ERR_INVALID_ARG;
  fprintf(f, "stage,index,begin_ms,end_ms\n");
  for (int s = 0; s < 8; ++s)
    for (size_t i = 0; i < c->prof_ev[s].size(); ++i) {
      float a = 0, b = 0;
      cudaEventElapsedTime(&a, ref, c->prof_ev[s][i].first);
      cudaEventElapsedTime(&b, ref, c->prof_ev[s][i].second);
      fprintf(f, "%d,%zu,%.4f,%.4f\n", s, i, a, b);
    }
  fclose(f);
  return ESVO_OK;
}
ESVO_API int esvo_profile_read(esvo_ctx* c, double ms[8], uint64_t cnt[8]) {
  CHECK_CTX(c);
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  for (int s = 0; s < 8; ++s) {
    double tot = 0;
    for (auto& pr : c->prof_ev[s]) {
      float t = 0;
      if (cudaEventElapsedTime(&t, pr.first, pr.second) == cudaSuccess) tot += t;
      c->prof_pool.push_back(pr.first); c->prof_pool.push_back(pr.second);
    }
    if (ms) ms[s] = tot;
    if (cnt) cnt[s] = c->prof_ev[s].size();
    c->prof_ev[s].clear();
  }
  return ESVO_OK;
}
ESVO_API int esvo_run_mapping(esvo_ctx* c) {
  CHECK_CTX(c);
  if (!c->obs_set) return ESVO_ERR_STATE;
  return run_mapping_frame(c);
}
ESVO_API int esvo_fetch_mapping_counters(esvo_ctx* c, uint64_t out[8]) {
  CHECK_CTX(c);
  return fetch_mapping_counters(c, out);
}
ESVO_API int esvo_mapping_at_time(esvo_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et, size_t n,
                                  const int64_t* pt, const double* poses, size_t np, uint64_t* counters) {
  int rc = esvo_stage_mapping_inputs(c, ex, ey, et, n, pt, poses, np);
  if (rc) return rc;
  if ((rc = esvo_run_mapping(c))) return rc;
  uint64_t ctr[8];
  if ((rc = fetch_mapping_counters(c, ctr))) return rc;   // also the sync that makes the caller's buffers reusable
  if (counters) std::memcpy(counters, ctr, sizeof(ctr));
  return ESVO_OK;
}

}  // extern "C"
