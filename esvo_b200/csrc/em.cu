// esvo_b200 product code -- the event-to-event matcher of the reference's comparison modes (sm_90a).
//
// Replaces esvo_core::core::EventMatcher::{createMatchProblem, match_all_HyperThread, match, match_an_event, warping2,
// patchInterpolation2, zncc_cost} (esvo_core/src/core/EventMatcher.cpp:51-346) as esvo_MVStereo drives it in its modes
// PURE_EVENT_MATCHING / EM_PLUS_ESTIMATION (esvo_core/src/esvo_MVStereo.cpp:257-266), and esvo_MVStereo::vEMP2vDP (:1072-1097).
//
// Design: one warp per left event.  The warp finds the event's temporal window in the time-ordered right events by binary
// search (toSec() doubles and ros::Time(double) rounding as the reference), then its lanes take the window's candidates 32
// at a time: polarity + time + epipolar checks read two LUT entries; a survivor (a few per event) is triangulated, warped
// into the time-surface pair and scored in-lane -- the two bilinear patches are evaluated on the fly in three passes (means,
// norms, correlation), so any patch size works without local arrays.  The lanes' best (cost, candidate) pairs meet in a
// lexicographic warp minimum, which is the reference's "first strictly smaller cost" rule.  Results are dense per event;
// em_order_kernel compacts them in the reference's thread-major order (same scheme as seeds_order_kernel, bm.cu).
// f64 throughout, no FMA contraction (-fmad=false).  A comparison harness, not a hot path: buffers are per call.
#include <cstdlib>
#include <vector>

#include "common.cuh"

namespace esvo {

__device__ int block_excl_scan(int v, int* s_warp, int& total);   // bm.cu

struct EmArgs {
  const uint16_t *lx, *ly; const int64_t* lt; const uint8_t* lp; int n;   // left events of all slices
  const int32_t* slice_of; const double* slice_poses;
  const uint16_t *rx, *ry; const int64_t* rt; const uint8_t* rp; int nr;  // right candidates, time-ordered
  const double *lut_l, *lut_r;
  const uint8_t *tl, *tr;                                                 // observation pair, row pitch dc.pitch
  double T_left_world[16];
  double time_thr, epi_thr, ncc_thr;
  int wx, wy, NT;
  int32_t *flag, *best_j; double *cost, *inv_depth;                       // dense per-event results
  unsigned long long* counters;                                           // [0] zncc evaluations, [1] matched events
};

// ros::Time(double): sec = floor(t), nsec = round((t - sec) * 1e9), normalised
__device__ __forceinline__ long long sec_to_ns_dev(double t) {
  long long sec = (long long)floor(t);
  long long nsec = llround(__dmul_rn(__dsub_rn(t, (double)sec), 1e9));
  sec += nsec / 1000000000LL; nsec %= 1000000000LL;
  return sec * 1000000000LL + nsec;
}

// patchInterpolation2 (:308-346) set-up: window origin and the four bilinear weights; false = outside the image
struct EmPatch { const uint8_t* base; double q1, q2, q3, q4; };
__device__ __forceinline__ bool em_patch_setup(const DevConsts& dc, const uint8_t* img, double x, double y, int wx, int wy, EmPatch& p) {
  const double fx = floor(x), fy = floor(y);
  const int ulx = (int)(fx - (wx - 1) / 2), uly = (int)(fy - (wy - 1) / 2);
  const int drx = (int)(fx + (wx - 1) / 2), dry = (int)(fy + (wy - 1) / 2);
  if (ulx < 0 || uly < 0) return false;
  if (drx >= dc.W || dry >= dc.H) return false;
  const int lo0 = (int)fy, lo1 = (int)fx;
  p.q1 = (lo1 + 1) - x; p.q2 = x - lo1; p.q3 = (lo0 + 1) - y; p.q4 = y - lo0;
  if (uly + wy >= dc.H || ulx + wx >= dc.W) return false;
  p.base = img + (size_t)uly * dc.pitch + ulx;
  return true;
}
__device__ __forceinline__ double em_patch_at(const EmPatch& p, int pitch, int yy, int xx) {
  const uint8_t* s0 = p.base + (size_t)yy * pitch + xx;
  const double r0 = p.q1 * (double)s0[0] + p.q2 * (double)s0[1];
  const double r1 = p.q1 * (double)s0[pitch] + p.q2 * (double)s0[pitch + 1];
  return p.q3 * r0 + p.q4 * r1;
}

// PerspectiveCamera::cam2World in the reference's literal form (4x4 cofactor inverse, fuse.cu).  Here and in
// seeds_to_points_kernel the point is re-projected right away: with an integral rectified coordinate and T_left_rv = I the
// re-projection sits exactly on a pixel boundary, so the last bit of p decides the patch's base pixel and the warp's border
// tests.  The closed form (x - cx - tx/z) z / fx rounds differently in about half of such warps; this path is not hot.
__device__ void cam2world_general(const DevConsts& dc, double x, double y, double rho, double& p0, double& p1, double& p2);   // fuse.cu

// warping2 (:276-306) + the two patchInterpolation2 + zncc_cost (:253-274) for one candidate depth
__device__ bool em_candidate_cost(const DevConsts& dc, const EmArgs& a, const double* T /*3x4, shared*/, double xl0, double xl1, double inv_depth,
                                  double& cost) {
  const int wx = a.wx, wy = a.wy;
  double p0, p1, p2;
  cam2world_general(dc, xl0, xl1, inv_depth, p0, p1, p2);
  double pl[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) pl[q] = T[q * 4 + 0] * p0 + T[q * 4 + 1] * p1 + T[q * 4 + 2] * p2 + T[q * 4 + 3];
  double h1[3], h2[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    h1[q] = dc.Pl[q * 4 + 0] * pl[0] + dc.Pl[q * 4 + 1] * pl[1] + dc.Pl[q * 4 + 2] * pl[2] + dc.Pl[q * 4 + 3];
    h2[q] = dc.Pr[q * 4 + 0] * pl[0] + dc.Pr[q * 4 + 1] * pl[1] + dc.Pr[q * 4 + 2] * pl[2] + dc.Pr[q * 4 + 3];
  }
  const double x1 = h1[0] / h1[2], y1 = h1[1] / h1[2], x2 = h2[0] / h2[2], y2 = h2[1] / h2[2];
  const int hx = (wx - 1) / 2, hy = (wy - 1) / 2, W = dc.W, H = dc.H;
  if (x1 < hx || x1 > W - hx || y1 < hy || y1 > H - hy) return false;
  if (x2 < hx || x2 > W - hx || y2 < hy || y2 > H - hy) return false;
  if (!(x1 == x1 && y1 == y1 && x2 == x2 && y2 == y2)) return false;        // NaN never passes the reference's comparisons either
  EmPatch A, B;
  if (!em_patch_setup(dc, a.tl, x1, y1, wx, wy, A)) return false;
  if (!em_patch_setup(dc, a.tr, x2, y2, wx, wy, B)) return false;
  const int pitch = dc.pitch;
  const double n = (double)(wx * wy);
  double sl = 0, sr = 0;
  for (int yy = 0; yy < wy; ++yy) for (int xx = 0; xx < wx; ++xx) { sl += em_patch_at(A, pitch, yy, xx); sr += em_patch_at(B, pitch, yy, xx); }
  const double ml = sl / n, mr = sr / n;
  double ql = 0, qr = 0;
  for (int yy = 0; yy < wy; ++yy) for (int xx = 0; xx < wx; ++xx) {
    const double u = em_patch_at(A, pitch, yy, xx) - ml, v = em_patch_at(B, pitch, yy, xx) - mr;
    ql += u * u; qr += v * v;
  }
  const double nl = sqrt(ql) + 1e-6, nr = sqrt(qr) + 1e-6;
  double s = 0;
  for (int yy = 0; yy < wy; ++yy) for (int xx = 0; xx < wx; ++xx)
    s += ((em_patch_at(A, pitch, yy, xx) - ml) / nl) * ((em_patch_at(B, pitch, yy, xx) - mr) / nr);
  cost = 0.5 * (1 - s);
  return true;
}

constexpr int EM_WARPS = 4;
__global__ void __launch_bounds__(EM_WARPS * 32) em_match_kernel(DevConsts dc, EmArgs a) {
  __shared__ double s_T[EM_WARPS][12];
  const unsigned FULLM = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * EM_WARPS + w;
  if (i >= a.n) return;
  // T_left_rv = inverse(T_world_left) * T_world_rv (:118-120), rows 0..2
  if (lane < 12) {
    const double* Tw = a.slice_poses + 16 * (size_t)a.slice_of[i];
    const int r = lane >> 2, cidx = lane & 3;
    double s = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += a.T_left_world[r * 4 + j] * Tw[j * 4 + cidx];
    s_T[w][lane] = s;
  }
  __syncwarp();
  // --- temporal check (:66-88)
  const double te = ns_to_sec_dev(a.lt[i]);
  const double lowS = ns_to_sec_dev(sec_to_ns_dev(te - a.time_thr / 2)), upS = ns_to_sec_dev(sec_to_ns_dev(te + a.time_thr / 2));
  int cb, ce;
  { int lo = 0, hi = a.nr; while (lo < hi) { const int mid = (lo + hi) >> 1; if (ns_to_sec_dev(a.rt[mid]) < lowS) lo = mid + 1; else hi = mid; } cb = lo; }
  { int lo = cb, hi = a.nr; while (lo < hi) { const int mid = (lo + hi) >> 1; if (ns_to_sec_dev(a.rt[mid]) < upS) lo = mid + 1; else hi = mid; } ce = lo; }
  const size_t li = (size_t)a.ly[i] * dc.W + a.lx[i];
  const double xl0 = a.lut_l[2 * li], xl1 = a.lut_l[2 * li + 1];
  const bool lpol = a.lp[i] != 0;
  const double bf = dc.baseline * dc.Pl[0];
  double my_cost = 1.0, my_depth = 0; int my_j = 0x7fffffff, my_first = 0x7fffffff, my_evals = 0;
  bool any_time = false;
  for (int base = cb; base < ce; base += 32) {
    const int j = base + lane;
    if (j < ce) {
      const double tj = ns_to_sec_dev(a.rt[j]);
      if (tj >= lowS && tj <= upS && ((a.rp[j] != 0) == lpol)) {
        any_time = true;
        // --- epipolar check (:93-108)
        const size_t ri = (size_t)a.ry[j] * dc.W + a.rx[j];
        const double xr0 = a.lut_r[2 * ri], xr1 = a.lut_r[2 * ri + 1];
        if (fabs(xl1 - xr1) <= a.epi_thr && xr0 < xl0) {
          if (j < my_first) my_first = j;
          // --- motion check (:110-150)
          const double disparity = xl0 - xr0;
          const double depth = bf / disparity;
          double cst;
          if (em_candidate_cost(dc, a, s_T[w], xl0, xl1, 1.0 / depth, cst)) {
            ++my_evals;
            if (cst < my_cost) { my_cost = cst; my_j = j; my_depth = depth; }     // candidates arrive in increasing j within a lane
          }
        }
      }
    }
  }
  // the reference scans the candidates in order and keeps the first strictly smaller cost = lexicographic minimum of (cost, j)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double oc = __shfl_xor_sync(FULLM, my_cost, o), od = __shfl_xor_sync(FULLM, my_depth, o);
    const int oj = __shfl_xor_sync(FULLM, my_j, o), of = __shfl_xor_sync(FULLM, my_first, o);
    if (oc < my_cost || (oc == my_cost && oj < my_j)) { my_cost = oc; my_j = oj; my_depth = od; }
    my_first = min(my_first, of);
    my_evals += __shfl_xor_sync(FULLM, my_evals, o);
  }
  any_time = __any_sync(FULLM, any_time);
  if (lane == 0) {
    int ok = 0, jb = 0; double c = 1.0, inv = 0;
    if (any_time && my_first != 0x7fffffff) {
      // min_cost stays 1.0 and best_match_id 0 / best_depth 0 when no candidate scored below 1 (:113-116,151)
      c = (my_j != 0x7fffffff) ? my_cost : 1.0;
      if (!(c > a.ncc_thr)) { ok = 1; jb = (my_j != 0x7fffffff) ? my_j : my_first; inv = 1.0 / ((my_j != 0x7fffffff) ? my_depth : 0.0); }
    }
    a.flag[i] = ok; a.best_j[i] = jb; a.cost[i] = c; a.inv_depth[i] = inv;
    if (my_evals) atomicAdd(&a.counters[0], (unsigned long long)my_evals);
  }
}

// virtual position v in the thread-major order -> event index (match(), :233-251)
__device__ __forceinline__ int em_tm_index(int v, int n, int NT) {
  int c = 0, start = 0;
  for (; c < NT; ++c) {
    const int members = (n > c) ? (n - c + NT - 1) / NT : 0;
    if (v < start + members) break;
    start += members;
  }
  return c + (v - start) * NT;
}
constexpr int kEmOrdBlock = 256;
__global__ void __launch_bounds__(kEmOrdBlock) em_order_kernel(DevConsts dc, EmArgs a, esvo_seed* out) {
  __shared__ int s_warp[33];
  __shared__ int s_base;
  const int n = a.n, NT = a.NT;
  const int v0 = blockIdx.x * kEmOrdBlock;
  if (v0 >= n) return;
  int pre = 0;
  for (int v = threadIdx.x; v < v0; v += kEmOrdBlock) pre += a.flag[em_tm_index(v, n, NT)];
  int tot_pre;
  block_excl_scan(pre, s_warp, tot_pre);
  if (threadIdx.x == 0) s_base = tot_pre;
  const int v = v0 + threadIdx.x;
  const int i = v < n ? em_tm_index(v, n, NT) : 0;
  const int f = v < n ? a.flag[i] : 0;
  int total;
  const int local = block_excl_scan(f, s_warp, total);
  const int pos = s_base + local;
  if (f) {
    esvo_seed s;
    s.x_left_raw[0] = (double)a.lx[i]; s.x_left_raw[1] = (double)a.ly[i];
    const size_t li = (size_t)a.ly[i] * dc.W + a.lx[i];
    s.x_left[0] = a.lut_l[2 * li]; s.x_left[1] = a.lut_l[2 * li + 1];
    const int j = a.best_j[i];
    const size_t ri = (size_t)a.ry[j] * dc.W + a.rx[j];
    s.x_right[0] = a.lut_r[2 * ri]; s.x_right[1] = a.lut_r[2 * ri + 1];
    s.t_ns = a.lt[i];
    const double* T = a.slice_poses + 16 * (size_t)a.slice_of[i];
#pragma unroll
    for (int q = 0; q < 16; ++q) s.T_world_virtual[q] = T[q];
    s.inv_depth = a.inv_depth[i]; s.cost = a.cost[i]; s.disp = s.x_left[0] - s.x_right[0];
    out[pos] = s;
  }
  if (v0 + kEmOrdBlock >= n && threadIdx.x == 0) a.counters[1] = (unsigned long long)(s_base + total);
}

// esvo_MVStereo::vEMP2vDP (esvo_MVStereo.cpp:1072-1097).  cam2World in the literal form (above): the SGM mode feeds integer
// pixel coordinates through here, whose re-projection sits exactly on a pixel boundary, so the last bit of p_cam decides
// which pixels the point lands on.
__global__ void seeds_to_points_kernel(DevConsts dc, const esvo_seed* __restrict__ seeds, int n, long long age, esvo_depth_point* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const esvo_seed& s = seeds[i];
  esvo_depth_point d;
  d.row = (int32_t)floor(s.x_left[1]); d.col = (int32_t)floor(s.x_left[0]);
  d.x[0] = s.x_left[0]; d.x[1] = s.x_left[1];
  d.inv_depth = s.inv_depth; d.scale2 = 0; d.nu = 0;
  d.variance = 1e-6;                                    // update(invDepth, 0) + boundVariance
  d.residual = s.cost; d.age = age;
  cam2world_general(dc, s.x_left[0], s.x_left[1], s.inv_depth, d.p_cam[0], d.p_cam[1], d.p_cam[2]);
#pragma unroll
  for (int q = 0; q < 16; ++q) d.T_world_cam[q] = s.T_world_virtual[q];
  out[i] = d;
}

// --------------------------------------------------------------------------------------------
// host launchers (synchronous; per-call buffers)
// --------------------------------------------------------------------------------------------
namespace {
struct DevBufs {   // frees everything it handed out
  std::vector<void*> p;
  ~DevBufs() { for (void* q : p) cudaFree(q); }
  template <class T> cudaError_t get(T** out, size_t n) { void* q = nullptr; cudaError_t e = cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T)); if (e == cudaSuccess) { p.push_back(q); *out = (T*)q; } return e; }
  template <class T> cudaError_t put(T** out, const T* src, size_t n, cudaStream_t st) {
    cudaError_t e = get(out, n);
    if (e == cudaSuccess && n) e = cudaMemcpyAsync(*out, src, n * sizeof(T), cudaMemcpyHostToDevice, st);
    return e;
  }
};
}  // namespace

int em_match(Ctx* c, const esvo_em_params* prm, const uint16_t* lx, const uint16_t* ly, const int64_t* lt, const uint8_t* lp, size_t nl,
             const int32_t* slice_counts, const double* slice_poses, size_t n_slices, const uint16_t* rx, const uint16_t* ry, const int64_t* rt,
             const uint8_t* rp, size_t nr, esvo_seed* out, size_t* n_seeds, uint64_t* n_evals) {
  std::vector<int32_t> slice_of;
  for (size_t s = 0; s < n_slices; ++s) slice_of.insert(slice_of.end(), (size_t)std::max(slice_counts[s], 0), (int32_t)s);
  const size_t total = std::min(slice_of.size(), nl);
  if (n_evals) *n_evals = 0;
  if (total == 0 || nr == 0) { *n_seeds = 0; return ESVO_OK; }
  if (total > 0x7fffff00u || nr > 0x7fffff00u) return ESVO_ERR_INVALID_ARG;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  DevBufs b;
  EmArgs a{};
  uint16_t *dlx, *dly, *drx, *dry; int64_t *dlt, *drt; uint8_t *dlp, *drp; int32_t* dso; double *dposes, *dlut_r; esvo_seed* dseeds;
  ESVO_CUDA_TRY(c, b.put(&dlx, lx, total, c->stream)); ESVO_CUDA_TRY(c, b.put(&dly, ly, total, c->stream));
  ESVO_CUDA_TRY(c, b.put(&dlt, lt, total, c->stream)); ESVO_CUDA_TRY(c, b.put(&dlp, lp, total, c->stream));
  ESVO_CUDA_TRY(c, b.put(&dso, slice_of.data(), total, c->stream)); ESVO_CUDA_TRY(c, b.put(&dposes, slice_poses, 16 * n_slices, c->stream));
  ESVO_CUDA_TRY(c, b.put(&drx, rx, nr, c->stream)); ESVO_CUDA_TRY(c, b.put(&dry, ry, nr, c->stream));
  ESVO_CUDA_TRY(c, b.put(&drt, rt, nr, c->stream)); ESVO_CUDA_TRY(c, b.put(&drp, rp, nr, c->stream));
  ESVO_CUDA_TRY(c, b.put(&dlut_r, c->cam[1].lut.data(), 2 * npix, c->stream));
  ESVO_CUDA_TRY(c, b.get(&a.flag, total)); ESVO_CUDA_TRY(c, b.get(&a.best_j, total));
  ESVO_CUDA_TRY(c, b.get(&a.cost, total)); ESVO_CUDA_TRY(c, b.get(&a.inv_depth, total));
  ESVO_CUDA_TRY(c, b.get(&a.counters, 2)); ESVO_CUDA_TRY(c, b.get(&dseeds, total));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(a.counters, 0, 16, c->stream));
  a.lx = dlx; a.ly = dly; a.lt = dlt; a.lp = dlp; a.n = (int)total; a.slice_of = dso; a.slice_poses = dposes;
  a.rx = drx; a.ry = dry; a.rt = drt; a.rp = drp; a.nr = (int)nr;
  a.lut_l = c->d_lut; a.lut_r = dlut_r;
  const SlotBufs& f = c->slot();
  a.tl = f.obs_l; a.tr = f.obs_r;      // EventMatcher::createMatchProblem does not smooth the observation (:51-58)
  std::memcpy(a.T_left_world, f.T_left_world_inv, sizeof(a.T_left_world));
  a.time_thr = prm->time_threshold_s; a.epi_thr = prm->epipolar_threshold; a.ncc_thr = prm->ts_ncc_threshold;
  a.wx = prm->patch_size_x; a.wy = prm->patch_size_y; a.NT = prm->num_thread < 1 ? 1 : prm->num_thread;
  em_match_kernel<<<div_up((int)total, EM_WARPS), EM_WARPS * 32, 0, c->stream>>>(c->dc, a);
  em_order_kernel<<<div_up((int)total, kEmOrdBlock), kEmOrdBlock, 0, c->stream>>>(c->dc, a, dseeds);
  c->launches += 2;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  unsigned long long h[2] = {0, 0};
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h, a.counters, 16, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (n_evals) *n_evals = h[0];
  const size_t cnt = (size_t)h[1];
  if (cnt > *n_seeds) { *n_seeds = cnt; return ESVO_ERR_CAPACITY; }
  if (cnt) ESVO_CUDA_TRY(c, cudaMemcpy(out, dseeds, cnt * sizeof(esvo_seed), cudaMemcpyDeviceToHost));
  *n_seeds = cnt;
  return ESVO_OK;
}

int seeds_to_points(Ctx* c, const esvo_seed* seeds, size_t n, esvo_depth_point* out) {
  if (n == 0) return ESVO_OK;
  DevBufs b;
  esvo_seed* ds; esvo_depth_point* dp;
  ESVO_CUDA_TRY(c, b.put(&ds, seeds, n, c->stream));
  ESVO_CUDA_TRY(c, b.get(&dp, n));
  seeds_to_points_kernel<<<div_up((int)n, 128), 128, 0, c->stream>>>(c->dc, ds, (int)n, (long long)c->prm.age_vis_threshold, dp);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(out, dp, n * sizeof(esvo_depth_point), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  return ESVO_OK;
}

}  // namespace esvo
