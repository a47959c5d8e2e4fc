// ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into or called from the product path.
//
// CPU restatement (f64, sequential) of the reference's time-surface raster and semi-dense
// stereo mapper.  Every function cites the reference file:line it follows
// (paths relative to /root/reference).
#pragma once
#include <deque>
#include <map>
#include <thread>

#include "eigen_lm.h"
#include "o_core.h"

namespace oracle {

// ---------------------------------------------------------------------------------------------
// Time surface: esvo_time_surface/include/esvo_time_surface/TimeSurface.h:28-96,
//               esvo_time_surface/src/TimeSurface.cpp:52-152,403-425
// ---------------------------------------------------------------------------------------------
struct Event { uint16_t x, y; int64_t ts; uint8_t pol; int64_t idx; };

struct TimeSurface {
  int W = 0, H = 0;
  size_t queueLen = 20;
  std::vector<std::deque<Event>> eq;   // EventQueueMat::eqMat_
  bool have_back = false;
  Event back{};                        // events_.back() after the insertion sort
  int64_t n_pushed = 0;
  std::vector<uint8_t> last_ts;        // last published image

  void init(int w, int h, int qlen) {
    W = w; H = h; queueLen = (size_t)qlen;
    eq.assign((size_t)W * H, {}); have_back = false; n_pushed = 0; last_ts.assign((size_t)W * H, 0);
  }
  // eventsCallback (TimeSurface.cpp:403-425): the insertion sort keeps events_ ordered by ts
  // (stable: an event goes after equal stamps), then pushes events_.back() -- the globally
  // latest event, which is `e` itself for time-ordered input -- into the per-pixel queue.
  void push(uint16_t x, uint16_t y, int64_t ts, uint8_t pol) {
    Event e{x, y, ts, pol, n_pushed++};
    if (!have_back || !(back.ts > e.ts)) { back = e; have_back = true; }
    const Event& last = back;
    // EventQueueMat::insertEvent (TimeSurface.h:39-50)
    if (last.x >= W || last.y >= H) return;
    auto& q = eq[(size_t)last.x + (size_t)W * last.y];
    q.push_back(last);
    q.back().idx = e.idx;   // the index grid reports the ARRIVAL that queued the entry (== last.idx for time-ordered input)
    while (q.size() > queueLen) q.pop_front();
  }
  // getMostRecentEventBeforeT (TimeSurface.h:52-75)
  bool mostRecentBefore(int x, int y, int64_t T, Event* ev) const {
    const auto& q = eq[(size_t)x + (size_t)W * y];
    for (auto it = q.rbegin(); it != q.rend(); ++it)
      if (it->ts < T) { *ev = *it; return true; }
    return false;
  }
  // createTimeSurfaceAtTime (TimeSurface.cpp:52-152)
  void build(int64_t T, const esvo_params& p, const Camera& cam, int64_t* idx_grid, uint8_t* out) {
    const double decay_sec = p.decay_ms / 1000.0;
    std::vector<double> map((size_t)W * H, 0.0);
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        Event ev;
        if (idx_grid) idx_grid[(size_t)y * W + x] = -1;
        if (!mostRecentBefore(x, y, T, &ev)) continue;
        if (!(ns_to_sec(ev.ts) > 0)) continue;  // :73
        if (idx_grid) idx_grid[(size_t)y * W + x] = ev.idx;
        const double dt = ns_to_sec(T - ev.ts);
        double polarity = ev.pol ? 1.0 : -1.0;
        double expVal = std::exp(-dt / decay_sec);
        if (!p.ignore_polarity) expVal *= polarity;
        if (p.time_surface_mode == ESVO_TS_BACKWARD) map[(size_t)y * W + x] = expVal;
        if (p.time_surface_mode == ESVO_TS_FORWARD) {  // :86-116
          double u = cam.lut[2 * ((size_t)y * W + x)], v = cam.lut[2 * ((size_t)y * W + x) + 1];
          if (u >= 0 && v >= 0) {
            size_t u_i = (size_t)std::floor(u), v_i = (size_t)std::floor(v);
            if (u_i + 1 < (size_t)W && v_i + 1 < (size_t)H) {
              double fu = u - u_i, fv = v - v_i, fu1 = 1.0 - fu, fv1 = 1.0 - fv;
              double* m = map.data();
              m[v_i * W + u_i] += fu1 * fv1 * expVal;
              m[v_i * W + u_i + 1] += fu * fv1 * expVal;
              m[(v_i + 1) * W + u_i] += fu1 * fv * expVal;
              m[(v_i + 1) * W + u_i + 1] += fu * fv * expVal;
              if (m[v_i * W + u_i] > 1) m[v_i * W + u_i] = 1;
              if (m[v_i * W + u_i + 1] > 1) m[v_i * W + u_i + 1] = 1;
              if (m[(v_i + 1) * W + u_i] > 1) m[(v_i + 1) * W + u_i] = 1;
              if (m[(v_i + 1) * W + u_i + 1] > 1) m[(v_i + 1) * W + u_i + 1] = 1;
            }
          }
        }
      }
    std::vector<uint8_t> img((size_t)W * H);
    for (size_t i = 0; i < img.size(); ++i) {
      double v = p.ignore_polarity ? 255.0 * map[i] : 255.0 * (map[i] + 1.0) / 2.0;  // :123-126
      img[i] = cvt_u8(v);                                                            // :127
    }
    if (p.median_blur_kernel_size > 0)                                               // :130-131
      median_blur_u8(img.data(), img.data(), W, H, 2 * p.median_blur_kernel_size + 1);
    if (p.time_surface_mode == ESVO_TS_BACKWARD) {                                   // :144-151
      std::vector<uint8_t> rect((size_t)W * H);
      remap_bilinear_u8(img.data(), rect.data(), W, H, cam.map1.data(), cam.map2.data());
      img.swap(rect);
    }
    last_ts = img;
    if (out) std::memcpy(out, img.data(), img.size());
  }
};

// ---------------------------------------------------------------------------------------------
// TimeSurfaceObservation (container/TimeSurfaceObservation.h)
// ---------------------------------------------------------------------------------------------
struct TsObs {
  int W = 0, H = 0;
  std::vector<uint8_t> img_left, img_right;   // cvImagePtr_left_/right_
  std::vector<double> TS_left, TS_right;      // cv2eigen -> f64 (row-major here)
  std::vector<double> TS_negative_left, dTS_negative_du_left, dTS_negative_dv_left;
  Mat4 tr = Mat4::identity();
  bool empty = true;
  void set(const uint8_t* l, const uint8_t* r, int w, int h) {
    W = w; H = h; size_t n = (size_t)W * H;
    img_left.assign(l, l + n); img_right.assign(r, r + n);
    TS_left.assign(n, 0); TS_right.assign(n, 0);
    for (size_t i = 0; i < n; ++i) { TS_left[i] = l[i]; TS_right[i] = r[i]; }
    empty = false;
  }
  // GaussianBlurTS (TimeSurfaceObservation.h:107-116)
  void GaussianBlurTS(int k) {
    size_t n = (size_t)W * H;
    std::vector<uint8_t> a(n), b(n);
    gaussian_blur_u8(img_left.data(), a.data(), W, H, k);
    gaussian_blur_u8(img_right.data(), b.data(), W, H, k);
    for (size_t i = 0; i < n; ++i) { TS_left[i] = a[i]; TS_right[i] = b[i]; }
  }
  // getTimeSurfaceNegative (:118-134)
  void getTimeSurfaceNegative(int k) {
    size_t n = (size_t)W * H;
    TS_negative_left.assign(n, 0);
    if (k > 0) {
      std::vector<uint8_t> a(n);
      gaussian_blur_u8(img_left.data(), a.data(), W, H, k);
      for (size_t i = 0; i < n; ++i) TS_negative_left[i] = 255.0 - (double)a[i];
    } else
      for (size_t i = 0; i < n; ++i) TS_negative_left[i] = 255.0 - TS_left[i];
  }
  // computeTsNegativeGrad (:136-147)
  void computeTsNegativeGrad() {
    size_t n = (size_t)W * H;
    dTS_negative_du_left.assign(n, 0); dTS_negative_dv_left.assign(n, 0);
    sobel3_f64(TS_negative_left.data(), dTS_negative_du_left.data(), dTS_negative_dv_left.data(), W, H);
  }
};

// patchInterpolation (DepthProblem.cpp:193-262; identical copy RegProblemLM.cpp:418-487).
// img row-major H x W; patch row-major wy x wx.
static inline bool patchInterpolation(const double* img, int W, int H, const double loc[2], int wx,
                                      int wy, double* patch) {
  int ulx = (int)(std::floor(loc[0]) - (wx - 1) / 2), uly = (int)(std::floor(loc[1]) - (wy - 1) / 2);
  int drx = (int)(std::floor(loc[0]) + (wx - 1) / 2), dry = (int)(std::floor(loc[1]) + (wy - 1) / 2);
  if (ulx < 0 || uly < 0) return false;
  if (drx >= W || dry >= H) return false;
  double di0 = loc[1], di1 = loc[0];
  int lo0 = (int)std::floor(di0), lo1 = (int)std::floor(di1);
  int up0 = lo0 + 1, up1 = lo1 + 1;
  double q1 = up1 - di1, q2 = di1 - lo1, q3 = up0 - di0, q4 = di0 - lo0;
  if (uly + wy >= H || ulx + wx >= W) return false;
  // R = q1*S[:, :wx] + q2*S[:, 1:]  (wy+1 rows);  patch = q3*R[:wy] + q4*R[1:]
  for (int y = 0; y < wy; ++y)
    for (int x = 0; x < wx; ++x) {
      const double* s0 = img + (size_t)(uly + y) * W + ulx + x;
      const double* s1 = s0 + W;
      double r0 = q1 * s0[0] + q2 * s0[1];
      double r1 = q1 * s1[0] + q2 * s1[1];
      patch[y * wx + x] = q3 * r0 + q4 * r1;
    }
  return true;
}

// ---------------------------------------------------------------------------------------------
// EventBM (core/EventBM.cpp)
// ---------------------------------------------------------------------------------------------
struct Seed {  // EventMatchPair
  double x_left_raw[2], x_left[2], x_right[2];
  int64_t t_ns; Mat4 trans; double invDepth, cost, disp;
};

struct EventBM {
  const CameraSystem* cs = nullptr;
  const TsObs* obs = nullptr;
  size_t wx = 15, wy = 7, min_disp = 1, max_disp = 40, step = 1;
  double thr = 0.1; bool updown = false;
  const double ZNCC_MAX = 1.0;
  uint64_t n_evals = 0;
  size_t coarseFail = 0, fineFail = 0, lowInfo = 0;

  // tools::meanStdDev / normalizePatch (utils.h:74-92); patches are wy x wx, traversed in Eigen's
  // storage order (column-major: x outer, y inner).
  static void normalizePatch(const double* src, double* dst, size_t n) {
    double sum = 0;
    for (size_t i = 0; i < n; ++i) sum += src[i];
    double mean = sum / n;
    double ss = 0;
    for (size_t i = 0; i < n; ++i) { double d = src[i] - mean; ss += d * d; }
    double sigma = std::sqrt(ss / n) + 1e-6;
    for (size_t i = 0; i < n; ++i) dst[i] = (src[i] - mean) / sigma;
  }
  // zncc_cost (EventBM.cpp:317-333)
  static double zncc_cost(const double* l, const double* r, size_t n) {
    double sl[256], sr[256];   // stack scratch for the usual 15x7 patch; heap only for larger ones
    std::vector<double> hl, hr;
    double *ln = sl, *rn = sr;
    if (n > 256) { hl.resize(n); hr.resize(n); ln = hl.data(); rn = hr.data(); }
    normalizePatch(l, ln, n);
    normalizePatch(r, rn, n);
    double s = 0;
    for (size_t i = 0; i < n; ++i) s += ln[i] * rn[i];
    return 0.5 * (1 - s / n);
  }
  // isValidPatch (:251-267)
  bool isValidPatch(int x, int y, int& ltx, int& lty) const {
    int hx = (int)((wx - 1) / 2), hy = (int)((wy - 1) / 2);
    ltx = x - hx; lty = y - hy;
    int rbx = x + hx, rby = y + hy;
    if (ltx < 1 || lty < 1 || rbx >= cs->left.W - 1 || rby >= cs->left.H - 1) return false;
    return true;
  }
  // block copy in column-major order (x outer, y inner) like Eigen's .block() of a MatrixXd
  void block(const std::vector<double>& img, int ltx, int lty, double* out) const {
    size_t k = 0;
    for (size_t x = 0; x < wx; ++x)
      for (size_t y = 0; y < wy; ++y) out[k++] = img[(size_t)(lty + y) * obs->W + ltx + x];
  }
  // epipolarSearching (:170-226)
  bool epipolarSearching(double& min_cost, int bestMatch[2], size_t& bestDisp, size_t start,
                         size_t end, size_t sstep, const int x1[2], const double* patch_src) {
    bool found = false;
    std::map<size_t, double> mDispCost;
    std::vector<double> patch_dst(wx * wy);
    for (size_t disp = start; disp <= end; disp += sstep) {
      int x2[2];
      if (!updown) { x2[0] = (int)(x1[0] - disp); x2[1] = x1[1]; }
      else { x2[0] = x1[0]; x2[1] = (int)(x1[1] - disp); }
      int ltx, lty;
      if (!isValidPatch(x2[0], x2[1], ltx, lty)) { mDispCost.emplace(disp, ZNCC_MAX); continue; }
      block(obs->TS_right, ltx, lty, patch_dst.data());
      double cost = zncc_cost(patch_src, patch_dst.data(), wx * wy);
      n_evals++;
      mDispCost.emplace(disp, cost);
      if (cost <= min_cost) { min_cost = cost; bestMatch[0] = x2[0]; bestMatch[1] = x2[1]; bestDisp = disp; }
    }
    if (sstep > 1) {
      if (mDispCost.find(bestDisp - sstep) != mDispCost.end() &&
          mDispCost.find(bestDisp + sstep) != mDispCost.end()) {
        if (mDispCost[bestDisp - sstep] < ZNCC_MAX && mDispCost[bestDisp + sstep] < ZNCC_MAX)
          if (min_cost < thr) found = true;
      }
    } else if (min_cost < thr) found = true;
    return found;
  }
  // match_an_event (:80-168).  poses sorted by stamp = StampTransformationMap.
  bool match_an_event(uint16_t ex, uint16_t ey, int64_t et, const int64_t* pose_t,
                      const double* poses, size_t n_poses, Seed& em) {
    const Camera& L = cs->left;
    size_t idx = (size_t)ey * L.W + ex;
    double xr[2] = {L.lut[2 * idx], L.lut[2 * idx + 1]};
    if (xr[0] < 0 || xr[0] > L.W - 1 || xr[1] < 0 || xr[1] > L.H - 1) return false;
    if (L.mask[(size_t)((long)xr[1]) * L.W + (size_t)((long)xr[0])] <= 125) return false;
    int x1[2] = {(int)std::floor(xr[0]), (int)std::floor(xr[1])};
    int ltx, lty;
    if (!isValidPatch(x1[0], x1[1], ltx, lty)) return false;
    std::vector<double> patch_src(wx * wy);
    block(obs->TS_left, ltx, lty, patch_src.data());
    size_t cnt = 0;
    for (double v : patch_src) cnt += (v < 1);
    if ((double)cnt > 0.95 * (double)patch_src.size()) { lowInfo++; return false; }
    double min_cost = ZNCC_MAX;
    int bestMatch[2] = {0, 0};
    size_t bestDisp = 0;
    if (!epipolarSearching(min_cost, bestMatch, bestDisp, min_disp, max_disp, step, x1, patch_src.data())) {
      coarseFail++; return false;
    }
    size_t fine_start = bestDisp - (step - 1);  // size_t arithmetic, ">= 0" is always true (:126)
    if (!epipolarSearching(min_cost, bestMatch, bestDisp, fine_start, bestDisp + (step - 1), 1, x1, patch_src.data())) {
      fineFail++; return false;
    }
    if (min_cost <= thr) {
      em.x_left_raw[0] = ex; em.x_left_raw[1] = ey;
      em.x_left[0] = xr[0]; em.x_left[1] = xr[1];
      em.x_right[0] = bestMatch[0]; em.x_right[1] = bestMatch[1];
      em.t_ns = et;
      double disparity = updown ? (double)(x1[1] - bestMatch[1]) : (double)(x1[0] - bestMatch[0]);
      double depth = cs->baseline * L.P[0] / disparity;
      // tools::StampTransformationMap_lower_bound (utils.h:64-69): compares toSec() doubles
      const double te = ns_to_sec(et);
      size_t lo = 0, hi = n_poses;
      while (lo < hi) { size_t mid = (lo + hi) / 2; if (ns_to_sec(pose_t[mid]) < te) lo = mid + 1; else hi = mid; }
      if (lo == n_poses) return false;
      em.trans = Mat4::from(poses + 16 * lo);
      em.invDepth = 1.0 / depth; em.cost = min_cost; em.disp = disparity;
      return true;
    }
    return false;
  }
  // match_all_HyperThread (:269-315): NT interleaved jobs, results concatenated per thread.
  // exec_threads > 1 only changes how the work is executed (timing legs); the output is always
  // assembled in the reference's NT-interleaved thread-major order.
  void match_all(const uint16_t* ex, const uint16_t* ey, const int64_t* et, size_t n,
                 const int64_t* pose_t, const double* poses, size_t n_poses, int NT,
                 std::vector<Seed>& vEMP, int exec_threads = 1) {
    vEMP.clear(); n_evals = 0;
    if (exec_threads <= 1) {
      for (int tid = 0; tid < NT; ++tid)
        for (size_t i = tid; i < n; i += NT) {
          Seed em;
          if (match_an_event(ex[i], ey[i], et[i], pose_t, poses, n_poses, em)) vEMP.push_back(em);
        }
      return;
    }
    std::vector<Seed> dense(n);
    std::vector<char> flag(n, 0);
    std::vector<uint64_t> ev(exec_threads, 0);
    std::vector<std::thread> th;
    for (int w = 0; w < exec_threads; ++w)
      th.emplace_back([&, w]() {
        EventBM me = *this;
        me.n_evals = 0;
        for (size_t i = w; i < n; i += exec_threads) flag[i] = me.match_an_event(ex[i], ey[i], et[i], pose_t, poses, n_poses, dense[i]);
        ev[w] = me.n_evals;
      });
    for (auto& t : th) t.join();
    for (auto e : ev) n_evals += e;
    for (int tid = 0; tid < NT; ++tid)
      for (size_t i = tid; i < n; i += NT) if (flag[i]) vEMP.push_back(dense[i]);
  }
};

// ---------------------------------------------------------------------------------------------
// DepthProblem (core/DepthProblem.cpp) + DepthProblemSolver (core/DepthProblemSolver.cpp)
// ---------------------------------------------------------------------------------------------
static thread_local uint64_t g_irls_iters = 0, g_irls_max = 0;  // diagnostics of the calling thread
static thread_local uint64_t g_irls_hist[8] = {0};  // non-degenerate evals by iteration count: <=4,<=8,<=16,<=32,<=64,<=256,<=1024,more
static thread_local uint64_t g_irls_nd_iters = 0, g_irls_deg = 0;
// TIMING AID ONLY (bench.py cpu_baseline.with_shortcut), default off so that parity stays literal: skip the reference's
// degenerate scale iteration the way the CUDA kernel does (lm.cu "degenerate regime": with m non-zero residuals and
// (nu+1) m / N < 0.95 the loop of DepthProblem.cpp:96 ends through sum == 0 -> scale = td_scale^2 wherever the guard proves
// that rounding at subnormal scales cannot pass its 5 % test first).
static int g_irls_shortcut = 0;
struct DepthProblem {
  const CameraSystem* cs = nullptr;
  const TsObs* obs = nullptr;
  int wx = 15, wy = 7, lsnorm = ESVO_LSNORM_TDIST;
  double td_nu = 0, td_scale = 0, td_scale2 = 0, td_stdvar = 0;
  double coor[2]; double T_left_virtual[12];  // 3x4
  mutable uint64_t n_evals = 0;

  void configure(const esvo_params& p) {
    wx = p.patch_size_x; wy = p.patch_size_y; lsnorm = p.lsnorm; td_nu = p.td_nu; td_scale = p.td_scale;
    td_scale2 = td_scale * td_scale;                    // pow(td_scale,2)   DepthProblem.h:33
    td_stdvar = std::sqrt(td_nu / (td_nu - 2) * td_scale2);  // DepthProblem.h:34
  }
  // setProblem (:17-32)
  void setProblem(const double c[2], const Mat4& T_world_virtual) {
    coor[0] = c[0]; coor[1] = c[1];
    Mat4 T_left_world = rigid_inverse(obs->tr);
    Mat4 T = mul(T_left_world, T_world_virtual);
    std::memcpy(T_left_virtual, T.m, 12 * sizeof(double));
  }
  // warping (:162-191)
  bool warping(double d, double x1[2], double x2[2]) const {
    double p_rv[3], pl[3];
    cs->left.cam2World(coor, d, p_rv);
    for (int i = 0; i < 3; ++i)
      pl[i] = T_left_virtual[i * 4 + 0] * p_rv[0] + T_left_virtual[i * 4 + 1] * p_rv[1] +
              T_left_virtual[i * 4 + 2] * p_rv[2] + T_left_virtual[i * 4 + 3];
    cs->left.world2Cam(pl, x1);
    cs->right.world2Cam(pl, x2);
    int width = cs->left.W, height = cs->left.H;
    if (x1[0] < (wx - 1) / 2 || x1[0] > width - (wx - 1) / 2 || x1[1] < (wy - 1) / 2 || x1[1] > height - (wy - 1) / 2) return false;
    if (x2[0] < (wx - 1) / 2 || x2[0] > width - (wx - 1) / 2 || x2[1] < (wy - 1) / 2 || x2[1] > height - (wy - 1) / 2) return false;
    return true;
  }
  void fill_invalid(double* fvec) const {  // :40-58, :140-157
    const int N = wx * wy;
    if (lsnorm == ESVO_LSNORM_L2) for (int i = 0; i < N; ++i) fvec[i] = 255;
    else if (lsnorm == ESVO_LSNORM_ZNCC) for (int i = 0; i < N; ++i) fvec[i] = 2 / std::sqrt((double)N);
    else for (int i = 0; i < N; ++i) {
      double residual = 255;
      double r = residual / td_scale;
      double weight = (td_nu + 1) / (td_nu + r * r);
      fvec[i] = std::sqrt(weight) * residual;
    }
  }
  // operator() (:34-160)
  int operator()(double rho, double* fvec) const {
    n_evals++;
    const int N = wx * wy;
    double x1[2], x2[2];
    if (!warping(rho, x1, x2)) { fill_invalid(fvec); return 0; }
    double st1[256], st2[256], sR[256], sR2[256];
    std::vector<double> h1, h2, h3, h4;
    double *tau1 = st1, *tau2 = st2, *vR = sR, *vR2 = sR2;
    if (N > 256) { h1.resize(N); h2.resize(N); h3.resize(N); h4.resize(N); tau1 = h1.data(); tau2 = h2.data(); vR = h3.data(); vR2 = h4.data(); }
    if (patchInterpolation(obs->TS_left.data(), obs->W, obs->H, x1, wx, wy, tau1) &&
        patchInterpolation(obs->TS_right.data(), obs->W, obs->H, x2, wx, wy, tau2)) {
      if (lsnorm == ESVO_LSNORM_L2) {
        for (int i = 0; i < N; ++i) fvec[i] = tau1[i] - tau2[i];
      } else if (lsnorm == ESVO_LSNORM_ZNCC) {
        double m1 = 0, m2 = 0;
        for (int i = 0; i < N; ++i) { m1 += tau1[i]; m2 += tau2[i]; }
        m1 /= N; m2 /= N;
        double s1 = 0, s2 = 0;
        for (int i = 0; i < N; ++i) { s1 += (tau1[i] - m1) * (tau1[i] - m1); s2 += (tau2[i] - m2) * (tau2[i] - m2); }
        s1 = std::sqrt(s1 / N) + 1e-6; s2 = std::sqrt(s2 / N) + 1e-6;
        for (int i = 0; i < N; ++i) fvec[i] = ((tau1[i] - m1) / s1 - (tau2[i] - m2) / s2) / std::sqrt((double)N);
      } else {
        double s1 = td_scale2, s2 = -1.0;
        bool first = true;
        uint64_t loc = 0;
        if (g_irls_shortcut) {
          int nzs = 0; double rmin = 1e300;
          for (int i = 0; i < N; ++i) { vR[i] = tau1[i] - tau2[i]; vR2[i] = vR[i] * vR[i]; if (vR[i] != 0) { nzs++; rmin = std::min(rmin, std::fabs(vR[i])); } }
          const double nu1 = td_nu + 1, gap = 0.95 * (double)N - nu1 * (double)nzs;   // the kernels' guard, DESIGN.md deviation 4
          if (nu1 * (double)nzs < 0.95 * (double)N * (1.0 - 1e-9) && gap * (rmin * rmin) >= 0x1p-49 * (double)N) { s2 = td_scale2; first = false; s1 = s2; }
        }
        while (std::fabs(s2 - s1) / s1 > 0.05 || first) {           // :96
          ++g_irls_iters; if (++loc > g_irls_max) g_irls_max = loc;
          if (!first) s1 = s2;
          double sum = 0;
          for (int i = 0; i < N; ++i) {
            if (first) { vR[i] = tau1[i] - tau2[i]; vR2[i] = vR[i] * vR[i]; }
            if (vR[i] != 0) sum += vR2[i] * (td_nu + 1) / (td_nu + vR2[i] / s1);
          }
          if (sum == 0) { s2 = td_scale2; break; }
          s2 = sum / N;
          first = false;
        }
        {
          int nz = 0; for (int i = 0; i < N; ++i) nz += (vR[i] != 0);
          if ((td_nu + 1) * nz < 0.95 * N) g_irls_deg++;
          else { g_irls_nd_iters += loc; int b = loc <= 4 ? 0 : loc <= 8 ? 1 : loc <= 16 ? 2 : loc <= 32 ? 3 : loc <= 64 ? 4 : loc <= 256 ? 5 : loc <= 1024 ? 6 : 7; g_irls_hist[b]++; }
        }
        for (int i = 0; i < N; ++i) {
          double weight = (td_nu + 1) / (td_nu + vR2[i] / s2);
          fvec[i] = std::sqrt(weight) * vR[i];
        }
      }
      return 1;
    }
    fill_invalid(fvec);
    return 0;
  }
};

struct DepthSolver {
  const CameraSystem* cs = nullptr;
  esvo_params prm;
  uint64_t n_evals = 0;

  // solve_single_problem_numerical (DepthProblemSolver.cpp:138-214)
  bool solve_single(double d_init, DepthProblem& dp, double result[3]) {
    const int m = dp.wx * dp.wy;
    LevenbergMarquardt lm;
    lm.f = [&](const std::vector<double>& x, std::vector<double>& fv) { dp(x[0], fv.data()); return 0; };
    lm.df = [&](const std::vector<double>& x, std::vector<double>& J) { return numerical_diff_forward(lm.f, x, J, m); };
    lm.ftol = 1e-6; lm.xtol = 1e-6; lm.maxfev = prm.max_iteration * 3;
    std::vector<double> x(1, d_init);
    if (lm.minimizeInit(x, m) == LM_ImproperInputParameters) return false;
    size_t iteration = 0; int state = 0;
    while (true) {
      LMStatus status = lm.minimizeOneStep(x);
      iteration++;
      if (iteration >= (size_t)prm.max_iteration) break;
      bool terminate = false;
      if (status == 2 || status == 3) { if (state == 0) state++; else terminate = true; }
      if (terminate) break;
    }
    if (x[0] <= 0.001) return false;
    result[0] = x[0];
    covar(lm.fjac, m, 1, lm.qrfac.perm);
    if (prm.lsnorm == ESVO_LSNORM_L2) {
      double fnorm = vnorm(lm.fvec.data(), m);
      double covfac = fnorm * fnorm / (m - 1);
      result[1] = covfac * lm.fjac[0];
    }
    if (prm.lsnorm == ESVO_LSNORM_TDIST) result[1] = (dp.td_stdvar * dp.td_stdvar) * lm.fjac[0];
    result[2] = lm.fnorm * lm.fnorm;
    return true;
  }
  // solve + solve_multiple_problems (:28-136), thread-major output order.
  void solve(const std::vector<Seed>& vEMP, const TsObs& obs, std::vector<DepthPoint>& vdp, int exec_threads = 1) {
    vdp.clear(); n_evals = 0;
    const int NT = prm.num_thread_mapping;
    DepthProblem dp; dp.cs = cs; dp.obs = &obs; dp.configure(prm);
    std::vector<double> dres; std::vector<char> dflag;
    if (exec_threads > 1) {  // timing legs: same results, solved by exec_threads threads
      dres.assign(3 * vEMP.size(), 0); dflag.assign(vEMP.size(), 0);
      std::vector<uint64_t> ev(exec_threads, 0);
      std::vector<std::thread> th;
      for (int w = 0; w < exec_threads; ++w)
        th.emplace_back([&, w]() {
          DepthSolver me = *this;
          DepthProblem q; q.cs = cs; q.obs = &obs; q.configure(prm);
          for (size_t i = w; i < vEMP.size(); i += exec_threads) {
            q.setProblem(vEMP[i].x_left, vEMP[i].trans);
            dflag[i] = me.solve_single(vEMP[i].invDepth, q, &dres[3 * i]);
          }
          ev[w] = q.n_evals;
        });
      for (auto& t : th) t.join();
      for (auto e : ev) n_evals += e;
    }
    for (int tid = 0; tid < NT; ++tid)
      for (size_t i = tid; i < vEMP.size(); i += NT) {
        const Seed& s = vEMP[i];
        double result[3];
        if (exec_threads > 1) {
          if (!dflag[i]) continue;
          result[0] = dres[3 * i]; result[1] = dres[3 * i + 1]; result[2] = dres[3 * i + 2];
        } else {
          dp.setProblem(s.x_left, s.trans);
          if (!solve_single(s.invDepth, dp, result)) continue;
        }
        DepthPoint d((int64_t)std::floor(s.x_left[1]), (int64_t)std::floor(s.x_left[0]));
        d.x[0] = s.x_left[0]; d.x[1] = s.x_left[1];
        cs->left.cam2World(s.x_left, result[0], d.p_cam);
        if (prm.lsnorm == ESVO_LSNORM_L2) d.update(result[0], result[1]);
        else {
          double scale2_rho = result[1] * (prm.td_nu - 2) / prm.td_nu;
          d.update_studentT(result[0], scale2_rho, result[1], prm.td_nu);
        }
        d.residual = result[2];
        d.T_world_cam = s.trans;
        vdp.push_back(d);
      }
    if (exec_threads <= 1) n_evals = dp.n_evals;
  }
  // pointCulling (:217-244)
  static void cull(std::vector<DepthPoint>& vdp, double std_thr, double cost_thr, double rmin, double rmax) {
    std::vector<DepthPoint> out;
    for (auto& d : vdp)
      if (d.variance <= std_thr * std_thr && d.residual <= cost_thr && d.valid() && d.invDepth >= rmin && d.invDepth <= rmax)
        out.push_back(d);
    vdp.swap(out);
  }
};

// ---------------------------------------------------------------------------------------------
// DepthMap (SmartGrid<DepthPoint>) with list-order semantics, DepthFusion, DepthRegularization
// ---------------------------------------------------------------------------------------------
struct DepthMap {
  int W = 0, H = 0;
  std::vector<int> grid;              // index into elems, -1 = NULL
  std::vector<DepthPoint> elems;      // insertion order (SmartGrid::_elements)
  std::vector<int> cell_of;           // true grid cell of each element (see DESIGN.md: the
                                      // reference keys erasure on the element's row_/col_, which
                                      // DepthFusion.cpp:186 may have overwritten -> UB there)
  std::vector<char> alive;
  void reset(int w, int h) { W = w; H = h; grid.assign((size_t)W * H, -1); elems.clear(); cell_of.clear(); alive.clear(); }
  bool exists(int r, int c) const { return grid[(size_t)r * W + c] >= 0; }
  DepthPoint& get(int r, int c) { return elems[grid[(size_t)r * W + c]]; }
  void set(int r, int c, const DepthPoint& v) {  // SmartGrid::set (:  copy without location)
    int& g = grid[(size_t)r * W + c];
    if (g < 0) { g = (int)elems.size(); elems.emplace_back(r, c); cell_of.push_back(r * W + c); alive.push_back(1); }
    elems[g].copy_from(v);
  }
  size_t size() const { size_t n = 0; for (char a : alive) n += a; return n; }
  // SmartGrid::clean (SmartGrid.h:222-243)
  void clean(double var_thr, double age_thr, double rmax, double rmin) {
    for (size_t i = 0; i < elems.size(); ++i)
      if (alive[i] && !elems[i].valid(var_thr, age_thr, rmax, rmin)) { alive[i] = 0; grid[cell_of[i]] = -1; }
    compact();
  }
  void compact() {
    std::vector<DepthPoint> e2; std::vector<int> c2;
    for (size_t i = 0; i < elems.size(); ++i) if (alive[i]) { grid[cell_of[i]] = (int)e2.size(); e2.push_back(elems[i]); c2.push_back(cell_of[i]); }
    elems.swap(e2); cell_of.swap(c2); alive.assign(elems.size(), 1);
  }
};

struct DepthFusion {
  const CameraSystem* cs = nullptr;
  int lsnorm = ESVO_LSNORM_TDIST;
  static bool boundaryCheck(double x, double y, size_t w, size_t h) { return !(x < 0 || x >= w || y < 0 || y >= h); }
  // propagate_one_point (DepthFusion.cpp:18-68)
  bool propagate_one_point(const DepthPoint& prior, DepthPoint& prop, const Mat4& T) const {
    double pp[3];
    for (int i = 0; i < 3; ++i) pp[i] = T(i, 0) * prior.p_cam[0] + T(i, 1) * prior.p_cam[1] + T(i, 2) * prior.p_cam[2] + T(i, 3);
    double xp[2];
    cs->left.world2Cam(pp, xp);
    if (!boundaryCheck(xp[0], xp[1], cs->left.W, cs->left.H)) return false;
    prop = DepthPoint((int64_t)std::floor(xp[1]), (int64_t)std::floor(xp[0]));
    prop.x[0] = xp[0]; prop.x[1] = xp[1];
    double invDepth = 1.0 / pp[2];
    double den = T(2, 0) * prior.p_cam[0] + T(2, 1) * prior.p_cam[1] + T(2, 3);
    den /= prior.p_cam[2];
    den += T(2, 2);
    double J = T(2, 2) / (den * den);
    if (lsnorm == ESVO_LSNORM_L2) { double var = J * J * prior.variance; prop.update(invDepth, var); }
    else {
      double s2 = J * J * prior.scale2, nu = prior.nu, var = nu / (nu - 2) * s2;
      prop.update_studentT(invDepth, s2, var, nu);
    }
    std::memcpy(prop.p_cam, pp, sizeof(pp));
    prop.residual = prior.residual; prop.age = prior.age;
    return true;
  }
  // fusion (:90-192)
  int fusion(const DepthPoint& prop, DepthMap& dm, int radius) const {
    int numFusion = 0;
    // 64-bit coordinates: a NaN re-projection passes boundaryCheck(double) and becomes row = col = 2^63 through x86-64's
    // double -> size_t conversion, which the per-pixel boundaryCheck below then rejects (never truncate it to 32 bits)
    int64_t rr[9], cc[9]; int n = 0;
    if (radius == 0) { for (int dy = 0; dy <= 1; ++dy) for (int dx = 0; dx <= 1; ++dx) { rr[n] = prop.row + dy; cc[n] = prop.col + dx; n++; } }
    else { for (int dy = -1; dy <= 1; ++dy) for (int dx = -1; dx <= 1; ++dx) { rr[n] = prop.row + dy; cc[n] = prop.col + dx; n++; } }
    for (int i = 0; i < n; ++i) {
      if (rr[i] < 0 || cc[i] < 0 || rr[i] >= cs->left.H || cc[i] >= cs->left.W) continue;  // size_t wrap == out of range
      int row = (int)rr[i], col = (int)cc[i];
      if (!dm.exists(row, col)) {
        DepthPoint nw(row, col);
        if (lsnorm == ESVO_LSNORM_L2) nw.update(prop.invDepth, prop.variance);
        else nw.update_studentT(prop.invDepth, prop.scale2, prop.variance, prop.nu);
        nw.residual = prop.residual; nw.age = prop.age;
        cs->left.cam2World(nw.x, prop.invDepth, nw.p_cam);
        dm.set(row, col, nw);
      } else {
        DepthPoint& cur = dm.get(row, col);
        bool compat;
        if (lsnorm == ESVO_LSNORM_L2) {  // chiSquareTest (:205-218)
          double d2 = (prop.invDepth - cur.invDepth) * (prop.invDepth - cur.invDepth);
          compat = (d2 / prop.variance + d2 / cur.variance) < 5.99;
        } else {                          // studentTCompatibleTest (:221-231)
          double s1 = std::sqrt(prop.variance), s2 = std::sqrt(cur.variance), diff = std::fabs(prop.invDepth - cur.invDepth);
          compat = diff < 2 * s1 || diff < 2 * s2;
        }
        if (compat) {
          if (lsnorm == ESVO_LSNORM_L2) cur.update(prop.invDepth, prop.variance);
          else cur.update_studentT(prop.invDepth, prop.scale2, prop.variance, prop.nu);
          cur.age++;
          cur.residual = std::min(cur.residual, prop.residual);
          cs->left.cam2World(cur.x, prop.invDepth, cur.p_cam);
          numFusion++;
        } else {
          if (cur.invDepth - 2 * std::sqrt(cur.variance) > prop.invDepth) continue;
          if (prop.variance < cur.variance && prop.residual < cur.residual) cur = prop;  // :186 (copies row_/col_/x_ too)
        }
      }
    }
    return numFusion;
  }
  // naive_propagate_one_point (:290-327): always the Gaussian update, whatever LSnorm is
  bool naive_propagate_one_point(const DepthPoint& prior, DepthPoint& prop, const Mat4& T) const {
    double pp[3];
    for (int i = 0; i < 3; ++i) pp[i] = T(i, 0) * prior.p_cam[0] + T(i, 1) * prior.p_cam[1] + T(i, 2) * prior.p_cam[2] + T(i, 3);
    double xp[2];
    cs->left.world2Cam(pp, xp);
    if (!boundaryCheck(xp[0], xp[1], cs->left.W, cs->left.H)) return false;
    prop = DepthPoint((int64_t)std::floor(xp[1]), (int64_t)std::floor(xp[0]));
    prop.x[0] = xp[0]; prop.x[1] = xp[1];
    double invDepth = 1.0 / pp[2];
    double den = T(2, 0) * prior.p_cam[0] + T(2, 1) * prior.p_cam[1] + T(2, 3);
    den /= prior.p_cam[2];
    den += T(2, 2);
    double J = T(2, 2) / (den * den);
    prop.update(invDepth, J * J * prior.variance);
    std::memcpy(prop.p_cam, pp, sizeof(pp));
    prop.residual = prior.residual; prop.age = prior.age;
    return true;
  }
  // naive_propagation (:232-288): nearest-wins z-buffer over the 2x2 neighbourhood, no fusion
  void naive_propagation(const std::vector<DepthPoint>& obs, DepthMap& dm, const Mat4& T_world_frame) const {
    Mat4 T_frame_world = rigid_inverse(T_world_frame);
    for (const auto& o : obs) {
      Mat4 T_frame_obs = mul(T_frame_world, o.T_world_cam);
      DepthPoint prop;
      if (!naive_propagate_one_point(o, prop, T_frame_obs)) continue;
      for (int dy = 0; dy <= 1; ++dy)
        for (int dx = 0; dx <= 1; ++dx) {
          const int64_t row64 = prop.row + dy, col64 = prop.col + dx;   // 64-bit: see fusion()
          if (row64 < 0 || col64 < 0 || row64 >= cs->left.H || col64 >= cs->left.W) continue;
          int row = (int)row64, col = (int)col64;
          if (!dm.exists(row, col)) {                       // case 1
            DepthPoint nw(row, col);
            nw.update(prop.invDepth, prop.variance);
            nw.residual = prop.residual; nw.age = prop.age;
            cs->left.cam2World(nw.x, prop.invDepth, nw.p_cam);
            dm.set(row, col, nw);
          } else {                                           // case 2
            DepthPoint& cur = dm.get(row, col);
            if (cur.invDepth > prop.invDepth) continue;      // the propagated point is farther
            if (prop.residual < cur.residual) cur = prop;    // (copies row_/col_/x_ too)
          }
        }
    }
  }
  // The part of esvo_Mapping::InitializationAtTime after the SGM call (esvo_Mapping.cpp:446-480) with
  // createEdgeMask(..., bUndistortEvents = true, radius = 0) (:1000-1044) inlined: one DepthPoint per event whose
  // rectified pixel carries a valid disparity in range.  disp16 = CV_16S fixed point (disparity * 16).
  void sgm_points(const int16_t* disp16, const uint16_t* ex, const uint16_t* ey, size_t n, const Mat4& T_world_cam, double rho_min,
                  double rho_max, double age0, std::vector<DepthPoint>& out) const {
    out.clear();
    const int W = cs->left.W, H = cs->left.H;
    const double var_SGM = std::pow(0.001, 2);
    for (size_t i = 0; i < n; ++i) {
      if (ex[i] >= W || ey[i] >= H) continue;
      const double* coor = &cs->left.lut[2 * ((size_t)ey[i] * W + ex[i])];     // getRectifiedUndistortedCoordinate
      const int xc = (int)std::floor(coor[0]), yc = (int)std::floor(coor[1]);
      if (xc < 0 || xc >= W || yc < 0 || yc >= H) continue;
      const double disp = disp16[(size_t)yc * W + xc] / 16.0;
      if (disp < 0) continue;
      DepthPoint dp(xc, yc);                                   // DepthPoint dp(x, y): the reference passes (x, y) as (row, col)
      dp.x[0] = xc * 1.0; dp.x[1] = yc * 1.0;
      const double invDepth = disp / (cs->left.P[0] * cs->baseline);
      if (invDepth < rho_min || invDepth > rho_max) continue;
      cs->left.cam2World(dp.x, invDepth, dp.p_cam);
      dp.update(invDepth, var_SGM);
      dp.residual = 0.0;
      dp.age = (int64_t)age0;
      dp.T_world_cam = T_world_cam;
      out.push_back(dp);
    }
  }
  // update (:71-87)
  int update(const std::vector<DepthPoint>& obs, DepthMap& dm, const Mat4& T_world_frame, int radius) const {
    int numFusion = 0;
    Mat4 T_frame_world = rigid_inverse(T_world_frame);
    for (const auto& o : obs) {
      Mat4 T_frame_obs = mul(T_frame_world, o.T_world_cam);
      DepthPoint prop;
      if (!propagate_one_point(o, prop, T_frame_obs)) continue;
      numFusion += fusion(prop, dm, radius);
    }
    return numFusion;
  }
};

// DepthRegularization::apply (DepthRegularization.cpp:19-110) incl. the int/size_t loop quirk of
// SmartGrid::getNeighbourhood (SmartGrid.h:367-386): row<radius or col<radius => no neighbours.
static inline void regularize(DepthMap& dm, const esvo_params& p) {
  const int radius = p.reg_radius;
  std::vector<double> newRho(dm.elems.size());
  for (size_t e = 0; e < dm.elems.size(); ++e) {
    const DepthPoint& it = dm.elems[e];
    newRho[e] = it.invDepth;
    if (!it.valid()) continue;
    const int row = dm.cell_of[e] / dm.W, col = dm.cell_of[e] % dm.W;
    std::vector<const DepthPoint*> nb;
    if (row >= radius && col >= radius)
      for (int r = row - radius; r <= row + radius; ++r)
        for (int c = col - radius; c <= col + radius; ++c)
          if (r >= 0 && r < dm.H && c >= 0 && c < dm.W && dm.exists(r, c) && dm.get(r, c).valid()) nb.push_back(&dm.get(r, c));
    bool isSet = false;
    if (nb.size() > (size_t)p.reg_min_neighbours) {
      std::vector<const DepthPoint*> close;
      for (auto* q : nb) {
        double diff = std::fabs(it.invDepth - q->invDepth);
        if (diff < 2.0 * std::sqrt(it.variance) || diff < 2.0 * std::sqrt(q->variance)) close.push_back(q);
      }
      if (close.size() > (size_t)p.reg_min_close_neighbours) {
        double mean = 0.0;
        if (p.lsnorm == ESVO_LSNORM_L2) {
          double tot = 0.0;
          for (auto* q : close) tot += 1.0 / q->variance;
          for (auto* q : close) mean += q->invDepth * (1.0 / q->variance) / tot;
        } else {
          double nu_post = close[0]->nu, rho_post = close[0]->invDepth, s2_post = close[0]->scale2;
          for (size_t i = 1; i < close.size(); ++i) {
            double nu_prior = nu_post, rho_prior = rho_post, s2_prior = s2_post;
            double nu_obs = close[i]->nu, rho_obs = close[i]->invDepth, s2_obs = close[i]->scale2;
            nu_post = std::min(nu_prior, nu_obs);
            rho_post = (s2_obs * rho_prior + s2_prior * rho_obs) / (s2_obs + s2_prior);
            double d = rho_prior - rho_obs;
            s2_post = (nu_post + (d * d) / (s2_prior + s2_obs)) / (nu_post + 1) * (s2_prior * s2_obs) / (s2_prior + s2_obs);
          }
          mean = rho_post;
        }
        newRho[e] = mean; isSet = true;
      }
    }
    if (!isSet) newRho[e] = -1.0;
  }
  for (size_t e = 0; e < dm.elems.size(); ++e) dm.elems[e].invDepth = newRho[e];
}

}  // namespace oracle
