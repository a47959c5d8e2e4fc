// ORACLE -- TEST INFRASTRUCTURE ONLY.
// C entry points of the CPU restatement; same signatures as include/esvo_b200.h with the prefix
// esvo_oracle_.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline/reference legs
// may load this library.  PARITY STATUS: the reference has no tests or golden vectors and cannot
// be compiled here (needs ROS/Eigen/OpenCV C++): "parity unpinned" against the reference binary
// itself.  What pins this restatement instead (DESIGN.md section 2): its third-party pieces against cv2 4.13,
// scipy's MINPACK and libc rand; closed-form KATs; and, stage by stage, INDEPENDENT numpy / Python
// re-derivations written from the reference sources (tests/indep_numpy.py, tests/indep_fusion.py:
// time surface, EventBM accept set and order, DepthProblem residual, solver output, fusion case
// analysis, clean, regularisation, window bookkeeping, tracking residual / Jacobian / LM step, EventMatcher).
#include <chrono>
#include <cstdio>
#include <deque>
#include <string>
#include <thread>

#include "o_tracking.h"
#include "o_event_matcher.h"

using namespace oracle;

struct esvo_oracle_ctx {
  CameraSystem cs;
  esvo_params prm;
  size_t dmin = 0, dmax = 0;
  TimeSurface ts[2];
  TsObs obs;
  EventBM bm;
  DepthSolver solver;
  DepthFusion fusor;
  DepthMap dmap;
  Mat4 T_world_frame = Mat4::identity();
  std::deque<std::vector<DepthPoint>> window;  // dqvDepthPoints_
  RegProblem reg;
  TsObs trk_obs;
  uint64_t counters[8] = {0};
  int exec_threads = 1;   // timing legs only; results do not depend on it
  std::string err;
};

#define OAPI extern "C" __attribute__((visibility("default")))

OAPI void esvo_oracle_default_params(esvo_params* p) { default_params(p); }

OAPI esvo_oracle_ctx* esvo_oracle_create(int, const esvo_calib* l, const esvo_calib* r,
                                         const esvo_params* p, int* status) {
  if (!l || !r || !p || l->width != r->width || l->height != r->height || l->width <= 0) {
    if (status) *status = ESVO_ERR_INVALID_ARG;
    return nullptr;
  }
  auto* c = new esvo_oracle_ctx();
  c->cs.init(*l, *r);
  c->prm = *p;
  clip_disparity(c->cs, c->prm, c->dmin, c->dmax);
  for (int i = 0; i < 2; ++i) c->ts[i].init(l->width, l->height, p->max_event_queue_len);
  c->bm.cs = &c->cs; c->solver.cs = &c->cs; c->fusor.cs = &c->cs; c->reg.cs = &c->cs;
  c->solver.prm = *p; c->fusor.lsnorm = p->lsnorm; c->reg.prm = *p; c->reg.init();
  c->dmap.reset(l->width, l->height);
  if (status) *status = ESVO_OK;
  return c;
}
OAPI void esvo_oracle_destroy(esvo_oracle_ctx* c) { delete c; }

OAPI int esvo_oracle_set_rectify_tables(esvo_oracle_ctx* c, int cam, const float* m1, const float* m2,
                                        const double* lut, const uint8_t* mask) {
  if (!c || cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  Camera& C = cam ? c->cs.right : c->cs.left;
  size_t n = (size_t)C.W * C.H;
  if (m1) C.map1.assign(m1, m1 + n);
  if (m2) C.map2.assign(m2, m2 + n);
  if (lut) C.lut.assign(lut, lut + 2 * n);
  if (mask) C.mask.assign(mask, mask + n);
  return ESVO_OK;
}
OAPI int esvo_oracle_get_rectify_tables(esvo_oracle_ctx* c, int cam, float* m1, float* m2, double* lut,
                                        uint8_t* mask) {
  if (!c || cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  Camera& C = cam ? c->cs.right : c->cs.left;
  size_t n = (size_t)C.W * C.H;
  if (m1) std::memcpy(m1, C.map1.data(), n * sizeof(float));
  if (m2) std::memcpy(m2, C.map2.data(), n * sizeof(float));
  if (lut) std::memcpy(lut, C.lut.data(), 2 * n * sizeof(double));
  if (mask) std::memcpy(mask, C.mask.data(), n);
  return ESVO_OK;
}
OAPI int esvo_oracle_get_derived(esvo_oracle_ctx* c, double out[4]) {
  DepthProblem dp; dp.configure(c->prm);
  out[0] = c->cs.baseline; out[1] = (double)c->dmin; out[2] = (double)c->dmax; out[3] = dp.td_stdvar;
  return ESVO_OK;
}

// ---- time surface ----
OAPI int esvo_oracle_ts_push_events(esvo_oracle_ctx* c, int cam, const uint16_t* x, const uint16_t* y,
                                    const int64_t* t, const uint8_t* pol, size_t n) {
  if (!c || cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  for (size_t i = 0; i < n; ++i) c->ts[cam].push(x[i], y[i], t[i], pol ? pol[i] : 1);
  return ESVO_OK;
}
OAPI int esvo_oracle_ts_build(esvo_oracle_ctx* c, int cam, int64_t T, int64_t* idx, uint8_t* out) {
  if (!c || cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  c->ts[cam].build(T, c->prm, cam ? c->cs.right : c->cs.left, idx, out);
  return ESVO_OK;
}
OAPI int esvo_oracle_ts_reset(esvo_oracle_ctx* c, int cam) {
  c->ts[cam].init(c->cs.left.W, c->cs.left.H, c->prm.max_event_queue_len);
  return ESVO_OK;
}

// ---- mapping ----
OAPI int esvo_oracle_set_ts_pair(esvo_oracle_ctx* c, const uint8_t* l, const uint8_t* r, const double T[16]) {
  const uint8_t* L = l ? l : c->ts[0].last_ts.data();
  const uint8_t* R = r ? r : c->ts[1].last_ts.data();
  c->obs.set(L, R, c->cs.left.W, c->cs.left.H);
  c->obs.tr = Mat4::from(T);
  return ESVO_OK;
}
static void seed_to_pod(const Seed& s, esvo_seed* o) {
  std::memcpy(o->x_left_raw, s.x_left_raw, 16); std::memcpy(o->x_left, s.x_left, 16);
  std::memcpy(o->x_right, s.x_right, 16); o->t_ns = s.t_ns;
  std::memcpy(o->T_world_virtual, s.trans.m, sizeof(s.trans.m));
  o->inv_depth = s.invDepth; o->cost = s.cost; o->disp = s.disp;
}
static Seed seed_from_pod(const esvo_seed& o) {
  Seed s; std::memcpy(s.x_left_raw, o.x_left_raw, 16); std::memcpy(s.x_left, o.x_left, 16);
  std::memcpy(s.x_right, o.x_right, 16); s.t_ns = o.t_ns; s.trans = Mat4::from(o.T_world_virtual);
  s.invDepth = o.inv_depth; s.cost = o.cost; s.disp = o.disp; return s;
}
static void bm_configure(esvo_oracle_ctx* c) {
  c->bm.obs = &c->obs; c->bm.wx = c->prm.patch_size_x; c->bm.wy = c->prm.patch_size_y;
  c->bm.min_disp = c->dmin; c->bm.max_disp = c->dmax; c->bm.step = c->prm.bm_step;
  c->bm.thr = c->prm.bm_zncc_threshold; c->bm.updown = c->prm.bm_updown != 0;
  if (c->prm.smooth_time_surface) c->obs.GaussianBlurTS(5);  // createMatchProblem (EventBM.cpp:68-72)
}
OAPI int esvo_oracle_bm_match(esvo_oracle_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et,
                              size_t n, const int64_t* pt, const double* poses, size_t np,
                              esvo_seed* out, size_t* n_seeds, uint64_t* n_evals) {
  if (!c || c->obs.empty) return ESVO_ERR_STATE;
  bm_configure(c);
  std::vector<Seed> v;
  c->bm.match_all(ex, ey, et, n, pt, poses, np, c->prm.num_thread_mapping, v);
  if (n_evals) *n_evals = c->bm.n_evals;
  if (v.size() > *n_seeds) { *n_seeds = v.size(); return ESVO_ERR_CAPACITY; }
  for (size_t i = 0; i < v.size(); ++i) seed_to_pod(v[i], out + i);
  *n_seeds = v.size();
  return ESVO_OK;
}
OAPI int esvo_oracle_depth_solve(esvo_oracle_ctx* c, const esvo_seed* seeds, size_t n, esvo_depth_point* out,
                                 size_t* n_out, uint64_t* n_evals) {
  if (!c || c->obs.empty) return ESVO_ERR_STATE;
  std::vector<Seed> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = seed_from_pod(seeds[i]);
  std::vector<DepthPoint> vdp;
  c->solver.solve(v, c->obs, vdp);
  if (n_evals) *n_evals = c->solver.n_evals;
  if (vdp.size() > *n_out) { *n_out = vdp.size(); return ESVO_ERR_CAPACITY; }
  for (size_t i = 0; i < vdp.size(); ++i) to_pod(vdp[i], out + i);
  *n_out = vdp.size();
  return ESVO_OK;
}
OAPI int esvo_oracle_depth_cull(esvo_oracle_ctx*, esvo_depth_point* pts, size_t* n, double std_thr, double cost_thr,
                                double rmin, double rmax) {
  std::vector<DepthPoint> v(*n);
  for (size_t i = 0; i < *n; ++i) v[i] = from_pod(pts[i]);
  DepthSolver::cull(v, std_thr, cost_thr, rmin, rmax);
  for (size_t i = 0; i < v.size(); ++i) to_pod(v[i], pts + i);
  *n = v.size();
  return ESVO_OK;
}
OAPI int esvo_oracle_fuse(esvo_oracle_ctx* c, const esvo_depth_point* pts, size_t n, const double T[16], int radius,
                          int reset_map, int* n_fusions) {
  if (reset_map) { c->dmap.reset(c->cs.left.W, c->cs.left.H); c->T_world_frame = Mat4::from(T); }
  std::vector<DepthPoint> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = from_pod(pts[i]);
  int nf = c->fusor.update(v, c->dmap, c->T_world_frame, radius);
  if (n_fusions) *n_fusions = nf;
  return ESVO_OK;
}
OAPI int esvo_oracle_map_clean(esvo_oracle_ctx* c, double var_thr, double age_thr, double rmax, double rmin) {
  c->dmap.clean(var_thr, age_thr, rmax, rmin);
  return ESVO_OK;
}
OAPI int esvo_oracle_map_regularize(esvo_oracle_ctx* c) { regularize(c->dmap, c->prm); return ESVO_OK; }
OAPI int esvo_oracle_map_download(esvo_oracle_ctx* c, esvo_depth_point* out, size_t* n) {
  size_t cnt = c->dmap.elems.size();
  if (cnt > *n) { *n = cnt; return ESVO_ERR_CAPACITY; }
  for (size_t i = 0; i < cnt; ++i) {
    to_pod(c->dmap.elems[i], out + i);
    std::memcpy(out[i].T_world_cam, c->T_world_frame.m, sizeof(c->T_world_frame.m));
  }
  *n = cnt;
  return ESVO_OK;
}
// InitializationAtTime (esvo_Mapping.cpp:433-492) downstream of the SGM call (the disparity map is an input).
OAPI int esvo_oracle_init_from_disparity(esvo_oracle_ctx* c, const int16_t* disp16, const uint16_t* ex, const uint16_t* ey, size_t n,
                                         const double T[16], size_t min_points, size_t* n_points, int* accepted) {
  if (!c || !disp16 || !T || (n && (!ex || !ey))) return ESVO_ERR_INVALID_ARG;
  c->dmap.reset(c->cs.left.W, c->cs.left.H);
  c->T_world_frame = Mat4::from(T);
  std::vector<DepthPoint> vdp;
  c->fusor.sgm_points(disp16, ex, ey, n, c->T_world_frame, c->prm.invdepth_min_range, c->prm.invdepth_max_range,
                      (double)c->prm.age_vis_threshold, vdp);
  if (n_points) *n_points = vdp.size();
  if (vdp.size() < min_points) { if (accepted) *accepted = 0; return ESVO_OK; }   // :481-483
  c->window.push_back(vdp);                                                        // :485
  c->fusor.naive_propagation(vdp, c->dmap, c->T_world_frame);                      // :486
  if (accepted) *accepted = 1;
  return ESVO_OK;
}
// ---- comparison modes of esvo_MVStereo (SURVEY 8f row 4) ----
// EventMatcher::createMatchProblem + match_all_HyperThread (EventMatcher.cpp:51-58,185-251) on the current observation pair
OAPI int esvo_oracle_em_match(esvo_oracle_ctx* c, const esvo_em_params* prm, const uint16_t* lx, const uint16_t* ly, const int64_t* lt,
                              const uint8_t* lp, size_t nl, const int32_t* slice_counts, const double* slice_poses, size_t n_slices,
                              const uint16_t* rx, const uint16_t* ry, const int64_t* rt, const uint8_t* rp, size_t nr, esvo_seed* out,
                              size_t* n_seeds, uint64_t* n_evals) {
  if (!c || !prm || !n_seeds || (nl && (!lx || !ly || !lt || !lp)) || (nr && (!rx || !ry || !rt || !rp)) || (n_slices && (!slice_counts || !slice_poses)))
    return ESVO_ERR_INVALID_ARG;
  if (c->obs.empty) return ESVO_ERR_STATE;
  EventMatcher em;
  em.cs = &c->cs; em.obs = &c->obs; em.NT = prm->num_thread < 1 ? 1 : prm->num_thread;
  em.time_thr = prm->time_threshold_s; em.epi_thr = prm->epipolar_threshold; em.ncc_thr = prm->ts_ncc_threshold;
  em.wx = prm->patch_size_x; em.wy = prm->patch_size_y;
  std::vector<Seed> v;
  em.match_all(lx, ly, lt, lp, nl, slice_counts, slice_poses, n_slices, rx, ry, rt, rp, nr, v);
  if (n_evals) *n_evals = em.n_evals;
  if (v.size() > *n_seeds) { *n_seeds = v.size(); return ESVO_ERR_CAPACITY; }
  for (size_t i = 0; i < v.size(); ++i) seed_to_pod(v[i], out + i);
  *n_seeds = v.size();
  return ESVO_OK;
}
// esvo_MVStereo::vEMP2vDP (esvo_MVStereo.cpp:1072-1097)
OAPI int esvo_oracle_seeds_to_points(esvo_oracle_ctx* c, const esvo_seed* seeds, size_t n, esvo_depth_point* out) {
  if (!c || (n && (!seeds || !out))) return ESVO_ERR_INVALID_ARG;
  std::vector<Seed> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = seed_from_pod(seeds[i]);
  std::vector<DepthPoint> vdp;
  vEMP2vDP(c->cs, v, (double)c->prm.age_vis_threshold, vdp);
  for (size_t i = 0; i < n; ++i) to_pod(vdp[i], out + i);
  return ESVO_OK;
}
// DepthFusion::naive_propagation (DepthFusion.cpp:232-288) of one vector into the ctx's DepthFrame
OAPI int esvo_oracle_naive_propagate(esvo_oracle_ctx* c, const esvo_depth_point* pts, size_t n, const double T[16], int reset_map) {
  if (!c || (n && !pts)) return ESVO_ERR_INVALID_ARG;
  if (reset_map) { if (!T) return ESVO_ERR_INVALID_ARG; c->dmap.reset(c->cs.left.W, c->cs.left.H); c->T_world_frame = Mat4::from(T); }
  std::vector<DepthPoint> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = from_pod(pts[i]);
  c->fusor.naive_propagation(v, c->dmap, c->T_world_frame);
  return ESVO_OK;
}
OAPI int esvo_oracle_ts_set_unordered_input(esvo_oracle_ctx*, int, int) { return ESVO_OK; }   // the literal port always handles it
OAPI int esvo_oracle_window_download(esvo_oracle_ctx* c, int index, esvo_depth_point* out, size_t* n) {
  if (!c || !n || index < 0 || (size_t)index >= c->window.size()) return ESVO_ERR_INVALID_ARG;
  const auto& v = c->window[(size_t)index];
  if (v.size() > *n) { *n = v.size(); return ESVO_ERR_CAPACITY; }
  for (size_t i = 0; i < v.size(); ++i) to_pod(v[i], out + i);
  *n = v.size();
  return ESVO_OK;
}
OAPI int esvo_oracle_set_irls_shortcut(int on) { g_irls_shortcut = on ? 1 : 0; return ESVO_OK; }   // timing aid, see o_mapping.h
OAPI int esvo_oracle_set_exec_threads(esvo_oracle_ctx* c, int n) { c->exec_threads = n < 1 ? 1 : n; return ESVO_OK; }
OAPI int esvo_oracle_mapping_reset(esvo_oracle_ctx* c) { c->window.clear(); return ESVO_OK; }

// MappingAtTime (esvo_Mapping.cpp:261-399) without the optional denoising mask (SURVEY 8f row 3).
OAPI int esvo_oracle_mapping_at_time(esvo_oracle_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et,
                                     size_t n, const int64_t* pt, const double* poses, size_t np,
                                     uint64_t* counters) {
  if (!c || c->obs.empty) return ESVO_ERR_STATE;
  const esvo_params& p = c->prm;
  c->dmap.reset(c->cs.left.W, c->cs.left.H);
  c->T_world_frame = c->obs.tr;
  bm_configure(c);
  std::vector<Seed> vEMP;
  c->bm.match_all(ex, ey, et, n, pt, poses, np, p.num_thread_mapping, vEMP, c->exec_threads);
  std::vector<DepthPoint> vdp;
  c->solver.solve(vEMP, c->obs, vdp, c->exec_threads);
  size_t n_solved = vdp.size();
  double cost_thr = p.residual_vis_threshold * p.residual_vis_threshold * (p.patch_size_x * p.patch_size_y);
  DepthSolver::cull(vdp, p.stdvar_vis_threshold, cost_thr, p.invdepth_min_range, p.invdepth_max_range);
  size_t n_culled = vdp.size();
  c->window.push_back(vdp);
  if (p.fusion_strategy == ESVO_FUSION_CONST_POINTS) {
    auto total = [&]() { size_t s = 0; for (auto& v : c->window) s += v.size(); return s; };
    while ((double)total() > 1.5 * p.max_num_fusion_points) c->window.pop_front();
  } else {
    while (c->window.size() > (size_t)p.max_num_fusion_frames) c->window.pop_front();
  }
  int nf = 0;
  for (auto it = c->window.rbegin(); it != c->window.rend(); ++it)
    nf += c->fusor.update(*it, c->dmap, c->T_world_frame, p.fusion_radius);
  if (c->window.size() >= (size_t)p.max_num_fusion_frames)
    c->dmap.clean(p.stdvar_vis_threshold * p.stdvar_vis_threshold, p.age_vis_threshold, p.invdepth_max_range,
                  p.invdepth_min_range);
  if (p.regularization) regularize(c->dmap, p);
  uint64_t ctr[8] = {n, vEMP.size(), n_solved, n_culled, (uint64_t)nf, c->bm.n_evals, c->solver.n_evals,
                     c->dmap.elems.size()};
  std::memcpy(c->counters, ctr, sizeof(ctr));
  if (counters) std::memcpy(counters, ctr, sizeof(ctr));
  return ESVO_OK;
}

// ---- tracking ----
OAPI int esvo_oracle_track_srand(esvo_oracle_ctx* c, unsigned seed) { c->reg.rng.seed(seed); return ESVO_OK; }
OAPI int esvo_oracle_track_reset(esvo_oracle_ctx* c, float* ref_xyz, size_t n, const double Twr[16],
                                 const double Twc[16], const uint8_t* ts_left) {
  if (c->prm.trk_patch_size_x != 1 || c->prm.trk_patch_size_y != 1) return ESVO_ERR_UNSUPPORTED;
  if (n < (size_t)c->prm.trk_batch_size) return 1;  // resetRegProblem (RegProblemSolverLM.cpp:52-57)
  const uint8_t* L = ts_left ? ts_left : c->ts[0].last_ts.data();
  c->trk_obs.set(L, L, c->cs.left.W, c->cs.left.H);
  c->reg.prm = c->prm;
  c->reg.n_evals = 0;
  c->reg.setProblem(ref_xyz, n, Mat4::from(Twr), Mat4::from(Twc), &c->trk_obs, true);
  return ESVO_OK;
}
OAPI int esvo_oracle_track_solve(esvo_oracle_ctx* c, int analytical, double Tout[16], esvo_lm_stats* st) {
  if (!c->reg.obs) return ESVO_ERR_STATE;
  int rc = c->reg.solve(analytical != 0, st);
  if (rc < 0) return ESVO_ERR_UNSUPPORTED;
  std::memcpy(Tout, c->reg.T_world_left.m, sizeof(double) * 16);
  return ESVO_OK;
}
OAPI int esvo_oracle_track_get_negative_ts(esvo_oracle_ctx* c, double* neg, double* du, double* dv) {
  size_t n = (size_t)c->cs.left.W * c->cs.left.H;
  if (c->trk_obs.TS_negative_left.size() != n) return ESVO_ERR_STATE;
  if (neg) std::memcpy(neg, c->trk_obs.TS_negative_left.data(), n * 8);
  if (du) std::memcpy(du, c->trk_obs.dTS_negative_du_left.data(), n * 8);
  if (dv) std::memcpy(dv, c->trk_obs.dTS_negative_dv_left.data(), n * 8);
  return ESVO_OK;
}

// Trace of the last esvo_oracle_track_solve (RegProblem::trace for the layout): copies up to cap doubles, *n = its length.
OAPI int esvo_oracle_track_trace(esvo_oracle_ctx* c, double* out, size_t cap, size_t* n) {
  if (!c || !n) return ESVO_ERR_INVALID_ARG;
  const auto& t = c->reg.trace;
  *n = t.size();
  if (t.size() > cap) return ESVO_ERR_CAPACITY;
  if (!t.empty()) std::memcpy(out, t.data(), t.size() * sizeof(double));
  return ESVO_OK;
}

// Pinning tap (tests/test_indep_pins.py): after esvo_oracle_track_reset, select batch 0 like the first solver iteration
// and return RegProblemLM::operator()(x) and df(0) for it, with the inputs an independent evaluation needs:
// pts (3 per point, ref frame), Rt = {R_ row-major (9), t_ (3)}.  fjac is row-major n x 6.  Returns the batch size.
static int track_eval_batch(esvo_oracle_ctx* c, size_t iteration, const double x[6], double* fvec, double* fjac, double* pts, double* Rt, int cap);
OAPI int esvo_oracle_op_track_eval(esvo_oracle_ctx* c, const double x[6], double* fvec, double* fjac, double* pts, double* Rt, int cap) {
  return track_eval_batch(c, 0, x, fvec, fjac, pts, Rt, cap);
}
// the same for the batch outer iteration `iteration` works on (RegProblemSolverLM.cpp:158-159), at the solver's CURRENT R_, t_
OAPI int esvo_oracle_op_track_eval_iter(esvo_oracle_ctx* c, int iteration, const double x[6], double* fvec, double* fjac, double* pts, double* Rt, int cap) {
  return track_eval_batch(c, (size_t)(iteration < 0 ? 0 : iteration), x, fvec, fjac, pts, Rt, cap);
}
static int track_eval_batch(esvo_oracle_ctx* c, size_t iteration, const double x[6], double* fvec, double* fjac, double* pts, double* Rt, int cap) {
  if (!c->reg.obs) return ESVO_ERR_STATE;
  c->reg.setStochasticSampling((iteration % c->reg.numBatches) * (size_t)c->prm.trk_batch_size, (size_t)c->prm.trk_batch_size);
  const int n = (int)c->reg.numPoints;
  if (n > cap) return ESVO_ERR_CAPACITY;
  std::vector<double> xv(x, x + 6), fv((size_t)n), J;
  if (c->reg.residuals(xv, fv) < 0) return ESVO_ERR_UNSUPPORTED;
  std::vector<double> x0(6, 0.0);
  if (c->reg.jacobian(x0, J) < 0) return ESVO_ERR_UNSUPPORTED;
  for (int i = 0; i < n; ++i) {
    fvec[i] = fv[(size_t)i];
    for (int j = 0; j < 6; ++j) fjac[i * 6 + j] = J[(size_t)j * n + i];
    for (int k = 0; k < 3; ++k) pts[3 * i + k] = c->reg.Sampled[3 * (size_t)i + k];
  }
  std::memcpy(Rt, c->reg.R_, 9 * sizeof(double)); std::memcpy(Rt + 9, c->reg.t_, 3 * sizeof(double));
  return n;
}

// ---- raw helpers exposed for pinning tests (cv2 / scipy / libc cross-checks) ----
OAPI void esvo_oracle_op_median3(const uint8_t* s, uint8_t* d, int W, int H, int k) { median_blur_u8(s, d, W, H, k); }
OAPI void esvo_oracle_op_remap_u8(const uint8_t* s, uint8_t* d, int W, int H, const float* mx, const float* my) { remap_bilinear_u8(s, d, W, H, mx, my); }
OAPI void esvo_oracle_op_gauss_u8(const uint8_t* s, uint8_t* d, int W, int H, int k) { gaussian_blur_u8(s, d, W, H, k); }
OAPI void esvo_oracle_op_sobel(const double* s, double* dx, double* dy, int W, int H) { sobel3_f64(s, dx, dy, W, H); }
OAPI void esvo_oracle_op_cvt_u8(const double* s, uint8_t* d, size_t n) { for (size_t i = 0; i < n; ++i) d[i] = cvt_u8(s[i]); }
OAPI int esvo_oracle_op_rand(unsigned seed, int* out, int n) { GlibcRand g; g.seed(seed); for (int i = 0; i < n; ++i) out[i] = g.next(); return 0; }
OAPI void esvo_oracle_op_polar(const double* M, double* Q) { polar_orthonormalize(M, Q); }
OAPI double esvo_oracle_op_zncc(const double* l, const double* r, size_t n) { return EventBM::zncc_cost(l, r, n); }
// Evaluate DepthProblem::operator() for one seed (fvec has patch_size_x*patch_size_y entries).
OAPI int esvo_oracle_op_depth_residual(esvo_oracle_ctx* c, const esvo_seed* s, double rho, double* fvec) {
  DepthProblem dp; dp.cs = &c->cs; dp.obs = &c->obs; dp.configure(c->prm);
  Seed sd = seed_from_pod(*s);
  dp.setProblem(sd.x_left, sd.trans);
  return dp(rho, fvec);
}
// The reference's solver loop for ONE seed (DepthProblemSolver.cpp:138-186, same statements as DepthSolver::solve_single)
// with a trace: trace[2k] = x after the k-th minimizeOneStep, trace[2k+1] = its status.  Returns the number of steps.
OAPI int esvo_oracle_op_depth_solve_trace(esvo_oracle_ctx* c, const esvo_seed* s, double* trace, int max_steps) {
  DepthProblem dp; dp.cs = &c->cs; dp.obs = &c->obs; dp.configure(c->prm);
  Seed sd = seed_from_pod(*s);
  dp.setProblem(sd.x_left, sd.trans);
  const int m = dp.wx * dp.wy;
  LevenbergMarquardt lm;
  lm.f = [&](const std::vector<double>& x, std::vector<double>& fv) { dp(x[0], fv.data()); return 0; };
  lm.df = [&](const std::vector<double>& x, std::vector<double>& J) { return numerical_diff_forward(lm.f, x, J, m); };
  lm.ftol = 1e-6; lm.xtol = 1e-6; lm.maxfev = c->prm.max_iteration * 3;
  std::vector<double> x(1, sd.invDepth);
  if (lm.minimizeInit(x, m) == LM_ImproperInputParameters) return -1;
  size_t iteration = 0; int state = 0, k = 0;
  while (true) {
    LMStatus status = lm.minimizeOneStep(x);
    if (k < max_steps) { trace[2 * k] = x[0]; trace[2 * k + 1] = (double)status; ++k; }
    iteration++;
    if (iteration >= (size_t)c->prm.max_iteration) break;
    bool terminate = false;
    if (status == 2 || status == 3) { if (state == 0) state++; else terminate = true; }
    if (terminate) break;
  }
  return k;
}
// Generic LM driver for pinning against MINPACK: minimise sum (a_i*exp(-b_i*x0)+x1*c_i - y_i)^2 style
// problems is done in Python; here we expose a scripted 1-D/2-D test function family:
//   f_i(x) = y_i - x0*exp(-x1*t_i)   (m points), forward-difference Jacobian, full convergence.
OAPI int esvo_oracle_op_lm_expfit(const double* t, const double* y, int m, double* x /*2*/, double ftol, double xtol,
                                  int maxfev, int max_steps, double* trace /*max_steps*2*/, int* nfev_out) {
  LevenbergMarquardt lm;
  lm.f = [&](const std::vector<double>& xx, std::vector<double>& fv) {
    for (int i = 0; i < m; ++i) fv[i] = y[i] - xx[0] * std::exp(-xx[1] * t[i]);
    return 0;
  };
  lm.df = [&](const std::vector<double>& xx, std::vector<double>& J) { return numerical_diff_forward(lm.f, xx, J, m); };
  lm.ftol = ftol; lm.xtol = xtol; lm.maxfev = maxfev;
  std::vector<double> xv = {x[0], x[1]};
  if (lm.minimizeInit(xv, m) == LM_ImproperInputParameters) return -100;
  int status = LM_Running, k = 0;
  while (k < max_steps) {
    status = lm.minimizeOneStep(xv);
    trace[2 * k] = xv[0]; trace[2 * k + 1] = xv[1]; ++k;
    if (status != LM_Running) break;
  }
  x[0] = xv[0]; x[1] = xv[1];
  if (nfev_out) *nfev_out = lm.nfev;
  return status * 1000 + k;
}

// ---- CPU baseline timing legs (bench.py cpu_baseline / --impl reference) ----
// Multi-threaded variants use the reference's own interleaved std::thread fan-out
// (EventBM.cpp:269-315, DepthProblemSolver.cpp:28-90) with NT threads.
OAPI double esvo_oracle_time_mapping(esvo_oracle_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et,
                                     size_t n, const int64_t* pt, const double* poses, size_t np, int NT, int reps,
                                     uint64_t* evals_out) {
  if (!c || c->obs.empty) return -1;
  bm_configure(c);
  uint64_t evals = 0;
  auto t0 = std::chrono::steady_clock::now();
  for (int rep = 0; rep < reps; ++rep) {
    std::vector<std::vector<Seed>> per(NT);
    std::vector<uint64_t> ev(NT, 0);
    {
      std::vector<std::thread> th;
      for (int tid = 0; tid < NT; ++tid)
        th.emplace_back([&, tid]() {
          EventBM bm = c->bm;  // per-thread counters
          bm.n_evals = 0;
          for (size_t i = tid; i < n; i += NT) {
            Seed em;
            if (bm.match_an_event(ex[i], ey[i], et[i], pt, poses, np, em)) per[tid].push_back(em);
          }
          ev[tid] = bm.n_evals;
        });
      for (auto& t : th) t.join();
    }
    std::vector<Seed> vEMP;
    for (auto& v : per) vEMP.insert(vEMP.end(), v.begin(), v.end());
    for (auto e : ev) evals += e;
    std::vector<std::vector<DepthPoint>> pv(NT);
    std::vector<uint64_t> ev2(NT, 0);
    {
      std::vector<std::thread> th;
      for (int tid = 0; tid < NT; ++tid)
        th.emplace_back([&, tid]() {
          DepthSolver sv = c->solver;
          DepthProblem dp; dp.cs = &c->cs; dp.obs = &c->obs; dp.configure(c->prm);
          for (size_t i = tid; i < vEMP.size(); i += NT) {
            const Seed& s = vEMP[i];
            dp.setProblem(s.x_left, s.trans);
            double result[3];
            if (!sv.solve_single(s.invDepth, dp, result)) continue;
            DepthPoint d((int64_t)std::floor(s.x_left[1]), (int64_t)std::floor(s.x_left[0]));
            d.invDepth = result[0]; d.variance = result[1]; d.residual = result[2];
            pv[tid].push_back(d);
          }
          ev2[tid] = dp.n_evals;
        });
      for (auto& t : th) t.join();
    }
    for (auto e : ev2) evals += e;
  }
  auto t1 = std::chrono::steady_clock::now();
  if (evals_out) *evals_out = evals;
  return std::chrono::duration<double>(t1 - t0).count();
}
OAPI double esvo_oracle_time_ts_build(esvo_oracle_ctx* c, int cam, int64_t T, int reps) {
  auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < reps; ++r) c->ts[cam].build(T, c->prm, cam ? c->cs.right : c->cs.left, nullptr, nullptr);
  auto t1 = std::chrono::steady_clock::now();
  return std::chrono::duration<double>(t1 - t0).count();
}
OAPI void esvo_oracle_op_irls_stats(uint64_t* out) { out[0] = g_irls_iters; out[1] = g_irls_max; g_irls_iters = 0; g_irls_max = 0; out[2] = g_irls_nd_iters; out[3] = g_irls_deg; for (int i = 0; i < 8; ++i) { out[4 + i] = g_irls_hist[i]; g_irls_hist[i] = 0; } g_irls_nd_iters = 0; g_irls_deg = 0; }
OAPI const char* esvo_oracle_version(void) { return "esvo-oracle 0.1 (CPU restatement, f64)"; }
