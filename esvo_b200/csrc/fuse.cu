// esvo_b200 product code -- depth propagation, Student-t fusion, map clean-up and regularisation
// (sm_90a).
//
// Replaces esvo_core::core::DepthFusion::{propagate_one_point, fusion, update, boundaryCheck,
// chiSquareTest, studentTCompatibleTest} (esvo_core/src/core/DepthFusion.cpp:18-231),
// DepthPoint::{update, update_studentT} (esvo_core/src/container/DepthPoint.cpp:145-188),
// SmartGrid::{set, clean, getNeighbourhood} (esvo_core/include/esvo_core/container/SmartGrid.h)
// and DepthRegularization::apply (esvo_core/src/core/DepthRegularization.cpp:19-110).
//
// The reference folds the propagated points into the map strictly one after another; the result
// at a pixel depends on the ORDER of the points that touch it, not on points touching other
// pixels.  So: (1) every point is propagated independently (one thread per point) and appends
// its 2x2 / 3x3 splat to a per-pixel linked list (one atomicExch per touched pixel);
// (2) one thread per pixel replays its own list in the global sequence order (list ids are the
// sequence numbers).  The map is a dense SoA over the image (the SmartGrid's element list order
// is kept as a "first touched" sequence number per pixel).
#include <algorithm>

#include "common.cuh"

namespace esvo {

struct MapSoA {
  uint8_t* exists;
  double *rho, *s2, *nu, *var, *res, *x0, *x1, *pc0, *pc1, *pc2, *rho_tmp;
  long long* age;
  int32_t *row, *col;
  unsigned long long* first_key;
};
struct FoldRec { double rho, s2, nu, var, res, sd2; };   // what the fold reads per contribution; sd2 = 2*sqrt(var)
struct PropSoA {  // propagated points staged for the current fold
  FoldRec* hot;
  uint8_t* ok;
  double *rho, *s2, *nu, *var, *res, *x0, *x1, *pc0, *pc1, *pc2;
  long long* age;
  int32_t *row, *col;
};
struct MapState {
  MapSoA m;
  PropSoA p;
  size_t prop_cap = 0, staged = 0;
  int32_t* head = nullptr;       // per pixel, -1 = empty
  int32_t* next = nullptr;       // per contribution (9 per staged point)
  int32_t* sort_pool = nullptr;  // ids of the long contribution lists, one segment per pixel (capacity = all contributions)
  int32_t* active = nullptr;     // pixels touched since the last reset, in first-touch order (count in d_scal[3])
  int32_t* pcnt = nullptr;       // contributions staged per pixel since its list was last folded (zeroed by the fold)
  int32_t* active_sorted = nullptr;  // the active pixels ordered by contribution count, longest first (fold_order_kernel)
  uint32_t* cbits = nullptr;     // one bit per contribution id: "this contribution created its pixel's element" (ordered hand-off)
  uint32_t* cprefix = nullptr;   // exclusive popcount prefix per word of cbits
  size_t cbits_words = 0;
  int folds = 0;                 // folds since the last reset
  size_t fold_words = 0;         // bitmap words covering the ids of the first fold after the reset
  bool list_valid = false;       // every existing pixel is in `active` (true from a reset until a kernel that ignores the list runs)
  bool cleaned = false;          // esvo_map_clean removed elements since the reset: their creator bits are stale
  unsigned long long seq_base = 0;
  double T_world_frame[16];
  double T_frame_world[16];
  esvo_depth_point* d_dl = nullptr;      // download staging
  unsigned long long* d_dl_keys = nullptr;
  unsigned long long* d_scal = nullptr;  // [0] n_fusions, [1] download count, [2] map size, [3] number of active pixels, [5] sort-pool cursor
  unsigned long long* h_scal = nullptr;
};

__device__ __forceinline__ void cam2world_f(const DevConsts& dc, double x, double y, double rho, double& p0, double& p1, double& p2) {
  const double z = 1.0 / rho;
  p0 = (x - dc.cx - dc.Pl[3] / z) * z / dc.fx;
  p1 = (y - dc.cy - dc.Pl[7] / z) * z / dc.fy;
  p2 = z * (1.0 - dc.Pl[11] / z);
}

// ---- stage: propagate_one_point (:18-68) + splat list insertion (:97-121) ----
// One launch covers up to FS_MAX vectors of the fusion window (newest first = sequence order).
constexpr int FS_MAX = 32;
struct FrameSet {
  const esvo_depth_point* pts[FS_MAX];
  const unsigned long long* cnt[FS_MAX];   // device counts (null = use cap)
  int cap[FS_MAX];
  int off[FS_MAX + 1];                     // thread / staging offsets (prefix sums of cap)
  int nframes;
};
struct Pose16 { double m[16]; };
__global__ void fuse_stage_kernel(DevConsts dc, FrameSet fs, Pose16 Tfw, int radius, int stage_off, PropSoA P, int32_t* head,
                                  int32_t* next, int32_t* active, int32_t* pcnt, unsigned long long* scal) {
  const double* T_frame_world = Tfw.m;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= fs.off[fs.nframes]) return;
  int f = 0;
  while (f + 1 < fs.nframes && t >= fs.off[f + 1]) ++f;
  const int j = t - fs.off[f];
  const int n = fs.cnt[f] ? (int)*fs.cnt[f] : fs.cap[f];
  const int sid = stage_off + t;
  if (j >= n) { P.ok[sid] = 0; return; }
  const esvo_depth_point& d = fs.pts[f][j];
  // T_frame_obs = T_frame_world * T_world_cam
  double T[12];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      double s = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) s += T_frame_world[r * 4 + k] * d.T_world_cam[k * 4 + c];
      T[r * 4 + c] = s;
    }
  double pp[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) pp[r] = T[r * 4] * d.p_cam[0] + T[r * 4 + 1] * d.p_cam[1] + T[r * 4 + 2] * d.p_cam[2] + T[r * 4 + 3];
  double h[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) h[r] = dc.Pl[r * 4] * pp[0] + dc.Pl[r * 4 + 1] * pp[1] + dc.Pl[r * 4 + 2] * pp[2] + dc.Pl[r * 4 + 3];
  const double xp = h[0] / h[2], yp = h[1] / h[2];
  const bool inb = !(xp < 0 || xp >= dc.W || yp < 0 || yp >= dc.H);  // boundaryCheck; NaN -> "inside" like the reference...
  if (!inb || !(xp == xp) || !(yp == yp)) { P.ok[sid] = 0; return; }  // ...but a NaN pixel index is UB there; drop it
  const int row = (int)floor(yp), col = (int)floor(xp);
  const double invDepth = 1.0 / pp[2];
  double den = T[8] * d.p_cam[0] + T[9] * d.p_cam[1] + T[11];
  den /= d.p_cam[2];
  den += T[10];
  const double J = T[10] / (den * den);
  P.ok[sid] = 1; P.row[sid] = row; P.col[sid] = col; P.x0[sid] = xp; P.x1[sid] = yp; P.rho[sid] = invDepth;
  if (dc.lsnorm == ESVO_LSNORM_L2) {
    double var = J * J * d.variance;
    if (var < 1e-6) var = 1e-6;  // DepthPoint::update -> boundVariance
    P.var[sid] = var; P.s2[sid] = 0; P.nu[sid] = 0;
  } else {
    const double s2 = J * J * d.scale2, nu = d.nu;
    P.s2[sid] = s2; P.nu[sid] = nu; P.var[sid] = nu / (nu - 2) * s2;
  }
  P.pc0[sid] = pp[0]; P.pc1[sid] = pp[1]; P.pc2[sid] = pp[2];
  P.res[sid] = d.residual; P.age[sid] = d.age;
  { FoldRec r; r.rho = invDepth; r.s2 = P.s2[sid]; r.nu = P.nu[sid]; r.var = P.var[sid]; r.res = d.residual; r.sd2 = 2 * sqrt(r.var); P.hot[sid] = r; }
  const int lo = radius == 0 ? 0 : -1;
  int i = 0;
  for (int dy = lo; dy <= 1; ++dy)
    for (int dx = lo; dx <= 1; ++dx, ++i) {
      const int r = row + dy, c = col + dx;
      if (r < 0 || c < 0 || r >= dc.H || c >= dc.W) continue;
      const int cid = sid * 9 + i;
      const int pix = r * dc.W + c;
      const int old = atomicExch(&head[pix], cid);
      next[cid] = old;
      atomicAdd(&pcnt[pix], 1);
      // first contribution to this pixel since its list was last folded: the pixel joins the active list (a pixel that
      // is folded twice between two resets is listed twice; the list kernels tolerate that, see map_*_list)
      if (old < 0) active[atomicAdd(&scal[3], 1ULL)] = pix;
    }
}

// ---- fold: DepthFusion::fusion (:123-190) replayed per pixel in sequence order ----
// NAIVE = DepthFusion::naive_propagation (:232-288): same ordered replay, but nearest-wins instead of fusion.
struct CleanArgs { int enable; double var_thr, age_thr, rmax, rmin; };

// ---- fold: DepthFusion::fusion (:123-190) replayed per pixel in sequence order ----
// The state of one map pixel while its contribution list is replayed.
struct FoldState {
  bool ex;
  double rho, s2, nu, var, res, x0, x1, pc0, pc1, pc2;
  long long age;
  int erow, ecol;
  unsigned long long fkey;
  int nfus;
  // p_cam is overwritten by every create / fuse step and never read back by the recurrence, so it is evaluated once at the
  // end from the inverse depth that set it last (pc_rho); a replacement copies the propagated p_cam.
  bool pc_pending;
  double pc_rho;
  double sdm;          // 2*sqrt(var) of the map point, refreshed whenever var changes
};
__device__ __forceinline__ void fold_load(const MapSoA& M, int pix, int row, int col, FoldState& f) {
  f.ex = M.exists[pix] != 0;
  f.rho = f.s2 = f.nu = f.var = f.res = f.x0 = f.x1 = f.pc0 = f.pc1 = f.pc2 = 0;
  f.age = 0; f.erow = row; f.ecol = col; f.fkey = 0; f.nfus = 0; f.pc_pending = false; f.pc_rho = 0;
  if (f.ex) {
    f.rho = M.rho[pix]; f.s2 = M.s2[pix]; f.nu = M.nu[pix]; f.var = M.var[pix]; f.res = M.res[pix]; f.x0 = M.x0[pix]; f.x1 = M.x1[pix];
    f.pc0 = M.pc0[pix]; f.pc1 = M.pc1[pix]; f.pc2 = M.pc2[pix]; f.age = M.age[pix]; f.erow = M.row[pix]; f.ecol = M.col[pix];
    f.fkey = M.first_key[pix];
  }
  f.sdm = f.ex ? 2 * sqrt(f.var) : 0.0;
}
// NAIVE = DepthFusion::naive_propagation (:232-288): same ordered replay, but nearest-wins instead of fusion.
template <bool NAIVE>
__device__ __forceinline__ void fold_apply(const DevConsts& dc, const PropSoA& P, FoldState& f, int row, int col, int cid, const FoldRec& r,
                                           unsigned long long seq_base) {
  const int sid = cid / 9;
  const double prho = r.rho, ps2 = r.s2, pnu = r.nu, pvar = r.var, pres = r.res;
  if (!f.ex) {  // case 1 (:126-145)
    f.ex = true; f.erow = row; f.ecol = col; f.x0 = col + 0.5; f.x1 = row + 0.5;
    f.rho = prho; f.var = pvar; f.s2 = ps2; f.nu = pnu;
    if (dc.lsnorm == ESVO_LSNORM_L2 && f.var < 1e-6) f.var = 1e-6;
    f.sdm = (dc.lsnorm == ESVO_LSNORM_L2) ? 2 * sqrt(f.var) : r.sd2;
    f.res = pres; f.age = P.age[sid];
    f.pc_rho = prho; f.pc_pending = true;
    f.fkey = seq_base + (unsigned long long)cid;
    if (NAIVE) { f.s2 = 0; f.nu = 0; }               // dp_new.update(): the Gaussian fields only
    return;
  }
  if (NAIVE) {                                       // case 2 of naive_propagation (:274-283)
    if (f.rho > prho) return;                        // the propagated point is farther
    if (pres < f.res) {                              // dm->get(row,col) = dp_prop
      f.rho = prho; f.s2 = ps2; f.nu = pnu; f.var = pvar; f.res = pres; f.age = P.age[sid];
      f.sdm = r.sd2;
      f.x0 = P.x0[sid]; f.x1 = P.x1[sid]; f.pc0 = P.pc0[sid]; f.pc1 = P.pc1[sid]; f.pc2 = P.pc2[sid];
      f.pc_pending = false;
      f.erow = P.row[sid]; f.ecol = P.col[sid];
    }
    return;
  }
  bool compat;
  if (dc.lsnorm == ESVO_LSNORM_L2) {
    const double d2 = (prho - f.rho) * (prho - f.rho);
    compat = (d2 / pvar + d2 / f.var) < 5.99;
  } else {
    const double diff = fabs(prho - f.rho);
    compat = diff < r.sd2 || diff < f.sdm;
  }
  if (compat) {  // case 2.1 (:162-177)
    bool fast_sqrt = false;
    if (!(f.rho > -1e-6)) {
      // DepthPoint::update / update_studentT take their "new point" branch for a map point that carries no valid inverse
      // depth (DepthPoint.cpp:158-163,181-187): overwrite, no inner age_++
      f.rho = prho; f.var = pvar; f.s2 = ps2; f.nu = pnu;
      if (dc.lsnorm == ESVO_LSNORM_L2 && f.var < 1e-6) f.var = 1e-6;
    } else if (dc.lsnorm == ESVO_LSNORM_L2) {
      const double t = f.rho;
      f.rho = (f.var * prho + pvar * t) / (f.var + pvar);
      const double tv = f.var;
      f.var = (tv * pvar) / (tv + pvar);
      if (f.var < 1e-6) f.var = 1e-6;
    } else {
      const double nu_u = fmin(pnu, f.nu);
      const double S = f.s2 + ps2;
      const double dd = f.rho - prho;
      if (S > 1e-200 && S < 1e200 && nu_u > 2.0 && nu_u < 1e15) {
        // the three divisions by S share one reciprocal; every quotient gets its own remainder correction (Markstein), i.e.
        // the correctly rounded value except for rare 1-ulp cases -- same arithmetic, a third of the dependent latency
        const double xr = rcp_nr(S);
        auto divS = [&](double a) { const double q = a * xr; return fma(fma(-S, q, a), xr, q); };
        const double rho_u = divS(ps2 * f.rho + f.s2 * prho);
        const double s2_u = divS(div_nr(nu_u + divS(dd * dd), nu_u + 1) * (f.s2 * ps2));
        f.rho = rho_u; f.s2 = s2_u; f.nu = nu_u + 1;
        f.var = div_nr(f.nu, f.nu - 2) * f.s2;
        f.age++;
        fast_sqrt = f.var > 1e-200 && f.var < 1e200;
      } else {
        const double rho_u = (ps2 * f.rho + f.s2 * prho) / S;
        const double s2_u = (nu_u + (dd * dd) / S) / (nu_u + 1) * (f.s2 * ps2) / S;
        f.rho = rho_u; f.s2 = s2_u; f.nu = nu_u + 1;
        f.var = f.nu / (f.nu - 2) * f.s2;
        f.age++;                                   // DepthPoint.cpp:179
      }
    }
    f.sdm = fast_sqrt ? 2 * sqrt_nr(f.var) : 2 * sqrt(f.var);
    f.age++;                                     // DepthFusion.cpp:171
    f.res = fmin(f.res, pres);
    f.pc_rho = prho; f.pc_pending = true;        // p_cam from the PROPAGATED rho (:174)
    f.nfus++;
  } else {       // case 2.2 (:178-188)
    if (f.rho - f.sdm > prho) return;
    if (pvar < f.var && pres < f.res) {              // dm->get(row,col) = dp_prop
      f.rho = prho; f.s2 = ps2; f.nu = pnu; f.var = pvar; f.res = pres; f.age = P.age[sid];
      f.sdm = r.sd2;
      f.x0 = P.x0[sid]; f.x1 = P.x1[sid]; f.pc0 = P.pc0[sid]; f.pc1 = P.pc1[sid]; f.pc2 = P.pc2[sid];
      f.pc_pending = false;
      f.erow = P.row[sid]; f.ecol = P.col[sid];
    }
  }
}
__device__ __forceinline__ void fold_store(const DevConsts& dc, MapSoA& M, int pix, FoldState& f, const CleanArgs& clean, uint32_t* cbits,
                                           unsigned long long seq_base, unsigned long long* scal) {
  if (f.pc_pending) cam2world_f(dc, f.x0, f.x1, f.pc_rho, f.pc0, f.pc1, f.pc2);
  // SmartGrid::clean (:222-243) right behind the fusion of the whole window (esvo_Mapping.cpp:385-386): the pixel's final state
  // is at hand, so the predicate is applied here instead of in a pass over the image
  if (clean.enable && f.ex && !(f.rho > -1e-6 && (double)f.age >= clean.age_thr && f.var <= clean.var_thr && f.rho <= clean.rmax && f.rho >= clean.rmin))
    f.ex = false;
  // creator bit of the surviving element: rank in the element list = number of set bits below it (map_gather_list_kernel)
  if (f.ex && cbits && f.fkey >= seq_base) { const unsigned long long cc = f.fkey - seq_base; atomicOr(&cbits[cc >> 5], 1u << (cc & 31)); }
  M.exists[pix] = f.ex ? 1 : 0;
  M.rho[pix] = f.rho; M.s2[pix] = f.s2; M.nu[pix] = f.nu; M.var[pix] = f.var; M.res[pix] = f.res; M.x0[pix] = f.x0; M.x1[pix] = f.x1;
  M.pc0[pix] = f.pc0; M.pc1[pix] = f.pc1; M.pc2[pix] = f.pc2; M.age[pix] = f.age; M.row[pix] = f.erow; M.col[pix] = f.ecol;
  M.first_key[pix] = f.fkey;
  if (f.nfus) atomicAdd(&scal[0], (unsigned long long)f.nfus);
}

// Thread-per-active-pixel form (dense over the active list): the production form (see fuse_finish for the measurement).
__device__ __forceinline__ void heap_sort_i32(int* ids, int cnt) {
  auto sift = [&](int start, int end) {
    int root = start;
    while (2 * root + 1 <= end) {
      int child = 2 * root + 1, sw = root;
      if (ids[sw] < ids[child]) sw = child;
      if (child + 1 <= end && ids[sw] < ids[child + 1]) sw = child + 1;
      if (sw == root) return;
      int tmp = ids[root]; ids[root] = ids[sw]; ids[sw] = tmp;
      root = sw;
    }
  };
  for (int st = (cnt - 2) / 2; st >= 0; --st) sift(st, cnt - 1);
  for (int end = cnt - 1; end > 0; --end) { int tmp = ids[end]; ids[end] = ids[0]; ids[0] = tmp; sift(0, end - 1); }
}
// Counting sort of the active pixels by their number of staged contributions, longest first (one block; a few thousand
// pixels).  A fold warp lives as long as the longest list among its 32 pixels: in first-touch order the sum of the per-warp
// maxima is 2.5x the sum in sorted order (13 140 vs 5 320 replay steps on the bench frame, ideal 5 230), and that warp-slot
// time is what the fold costs the frame pipeline.  Launching the longest lists first also shortens the kernel's tail.
__global__ void __launch_bounds__(1024) fold_order_kernel(const int32_t* __restrict__ active, const int32_t* __restrict__ pcnt,
                                                          unsigned long long* __restrict__ scal, int32_t* __restrict__ sorted) {
  __shared__ int s_hist[256], s_base[256];
  const int n = (int)scal[3];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&s_hist[min(pcnt[active[i]], 255)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int b = 255; b >= 0; --b) { s_base[b] = run; run += s_hist[b]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int pix = active[i];
    sorted[atomicAdd(&s_base[min(pcnt[pix], 255)], 1)] = pix;
  }
}
// ids of one pixel's contributions -> sequence order.  (The walk order is NOT close to sorted: an "reverse + insertion sort"
// variant was slower than the heap sort.)
// Lists of up to 64 ids go through a bitonic NETWORK held in registers (compile-time indices: 240 / 672 compare-exchanges of
// two instructions each, no memory traffic, no data-dependent branches); the local array is only the hand-over format of the
// list walk before and of the replay after.  Longer lists keep the heap sort.
template <int N>
__device__ __forceinline__ void network_sort_local(int* ids, int cnt) {
  int v[N];
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = i < cnt ? ids[i] : 0x7fffffff;
#pragma unroll
  for (int k = 2; k <= N; k <<= 1)
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1)
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const int l = i ^ j;
        if (l > i) {
          const int a = v[i], b = v[l];
          const int lo = min(a, b), hi = max(a, b);
          if ((i & k) == 0) { v[i] = lo; v[l] = hi; } else { v[i] = hi; v[l] = lo; }
        }
      }
#pragma unroll
  for (int i = 0; i < N; ++i) if (i < cnt) ids[i] = v[i];
}
// Lists longer than the local array (dense scenes; the 640x480 rig with fusion radius 1): kept out of line so that its
// registers do not count against the common path.
template <bool NAIVE>
__device__ __noinline__ void fold_long_list(const DevConsts& dc, const PropSoA& P, FoldState& f, int row, int col, int h, int total,
                                            const int32_t* __restrict__ next, int32_t* sort_pool, unsigned long long* scal,
                                            unsigned long long seq_base) {
  int* seg = sort_pool + atomicAdd(&scal[5], (unsigned long long)total);
  int k = 0;
  for (int q = h; q >= 0; q = next[q]) seg[k++] = q;
  heap_sort_i32(seg, total);
  FoldRec cur = P.hot[seg[0] / 9];
  for (int a = 0; a < total; ++a) {
    FoldRec nxt = cur;
    if (a + 1 < total) nxt = P.hot[seg[a + 1] / 9];
    fold_apply<NAIVE>(dc, P, f, row, col, seg[a], cur, seq_base);
    cur = nxt;
  }
}
template <bool NAIVE>
__global__ void fuse_fold_kernel(DevConsts dc, MapSoA M, PropSoA P, int32_t* head, const int32_t* __restrict__ next,
                                 const int32_t* __restrict__ active, int32_t* pcnt, unsigned long long seq_base, unsigned long long* scal,
                                 uint32_t* cbits, CleanArgs clean, int32_t* sort_pool) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if ((unsigned long long)t >= scal[3]) return;
  const int pix = active[t];
  int h = head[pix];
  if (h < 0) return;               // listed twice: the first copy folded it
  head[pix] = -1;
  pcnt[pix] = 0;
  // The list is in reverse insertion order of the atomics, not in sequence order: collect and sort.
  constexpr int CAP = 192;
  int ids[CAP];
  int cnt = 0, total = 0;
  for (int q = h; q >= 0; q = next[q]) { if (cnt < CAP) ids[cnt++] = q; ++total; }
  const int row = pix / dc.W, col = pix - row * dc.W;
  FoldState f;
  fold_load(M, pix, row, col, f);
  if (total <= CAP && cnt > 64) {
    // 65..192 ids: up to three runs of 64, each sorted by the register network, merged on the fly by the replay (the head
    // of every run is compared per step) -- no heap sort in local memory (0.13 of the 0.33 ms the fusion stage takes alone)
    const int e0 = 64, e1 = min(cnt, 128), e2 = cnt;
    network_sort_local<64>(ids, 64);
    network_sort_local<64>(ids + 64, e1 - 64);
    if (cnt > 128) network_sort_local<64>(ids + 128, e2 - 128);
    int h0 = 0, h1 = 64, h2 = 128;
    auto pop = [&]() -> int {
      int best = 0x7fffffff, which = 0;
      if (h0 < e0) best = ids[h0];
      if (h1 < e1) { const int v = ids[h1]; if (v < best) { best = v; which = 1; } }
      if (h2 < e2) { const int v = ids[h2]; if (v < best) { best = v; which = 2; } }
      if (which == 0) ++h0; else if (which == 1) ++h1; else ++h2;
      return best;
    };
    int id_cur = pop();
    FoldRec cur = P.hot[id_cur / 9];
    for (int a = 0; a < cnt; ++a) {
      int id_nxt = id_cur;
      FoldRec nxt = cur;
      if (a + 1 < cnt) { id_nxt = pop(); nxt = P.hot[id_nxt / 9]; }
      fold_apply<NAIVE>(dc, P, f, row, col, id_cur, cur, seq_base);
      id_cur = id_nxt; cur = nxt;
    }
  } else if (total <= CAP) {
    if (cnt <= 32) network_sort_local<32>(ids, cnt);
    else network_sort_local<64>(ids, cnt);
    FoldRec cur = P.hot[ids[0] / 9];
    for (int a = 0; a < cnt; ++a) {              // the next record is in flight while this one is folded
      FoldRec nxt = cur;
      if (a + 1 < cnt) nxt = P.hot[ids[a + 1] / 9];
      fold_apply<NAIVE>(dc, P, f, row, col, ids[a], cur, seq_base);
      cur = nxt;
    }
  } else {
    // long list (dense scenes: several hundred contributions on one pixel): its ids go to a private segment of the sort pool
    // (the pool holds one int per contribution, so the segments of all pixels always fit), heap-sorted there, replayed as above
    fold_long_list<NAIVE>(dc, P, f, row, col, h, total, next, sort_pool, scal, seq_base);
  }
  fold_store(dc, M, pix, f, clean, cbits, seq_base, scal);
}

// ---- SmartGrid::clean (:222-243) ----
__global__ void map_clean_kernel(int npix, MapSoA M, double var_thr, double age_thr, double rmax, double rmin) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix || !M.exists[pix]) return;
  const double rho = M.rho[pix];
  const bool valid = rho > -1e-6 && (double)M.age[pix] >= age_thr && M.var[pix] <= var_thr && rho <= rmax && rho >= rmin;
  if (!valid) M.exists[pix] = 0;
}

// ---- DepthRegularization::apply ----
// Thread per image pixel: any map (map_regularize_warp_kernel needs every existing pixel listed, i.e. one fold since the reset)
__global__ void map_regularize_kernel(DevConsts dc, MapSoA M, int radius, int min_nb, int min_close) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= dc.W * dc.H) return;
  if (!M.exists[pix]) return;
  const double rho = M.rho[pix];
  M.rho_tmp[pix] = rho;
  if (!(rho > -1e-6)) return;
  const int row = pix / dc.W, col = pix - row * dc.W;
  const double sig = 2.0 * sqrt(M.var[pix]);
  bool isSet = false;
  double mean = 0;
  // SmartGrid::getNeighbourhood's int/size_t loop never runs when row<radius or col<radius (SmartGrid.h:373-375)
  if (row >= radius && col >= radius) {
    int nb = 0, nclose = 0;
    double nu_post = 0, rho_post = 0, s2_post = 0, tot = 0;
    // pass 1: counts (+ l2 total inverse variance)
    for (int r = row - radius; r <= row + radius; ++r) {
      if (r >= dc.H) break;
      for (int c = col - radius; c <= col + radius; ++c) {
        if (c >= dc.W) break;
        const int q = r * dc.W + c;
        if (!M.exists[q]) continue;
        const double qr = M.rho[q];
        if (!(qr > -1e-6)) continue;
        nb++;
        const double diff = fabs(rho - qr);
        if (diff < sig || diff < 2.0 * sqrt(M.var[q])) {
          if (dc.lsnorm == ESVO_LSNORM_L2) tot += 1.0 / M.var[q];
          else if (nclose == 0) { nu_post = M.nu[q]; rho_post = qr; s2_post = M.s2[q]; }
          else {
            const double nu_prior = nu_post, rho_prior = rho_post, s2_prior = s2_post;
            const double nu_obs = M.nu[q], rho_obs = qr, s2_obs = M.s2[q];
            nu_post = fmin(nu_prior, nu_obs);
            rho_post = (s2_obs * rho_prior + s2_prior * rho_obs) / (s2_obs + s2_prior);
            const double d = rho_prior - rho_obs;
            s2_post = (nu_post + (d * d) / (s2_prior + s2_obs)) / (nu_post + 1) * (s2_prior * s2_obs) / (s2_prior + s2_obs);
          }
          nclose++;
        }
      }
    }
    if (nb > min_nb && nclose > min_close) {
      if (dc.lsnorm == ESVO_LSNORM_L2) {
        for (int r = row - radius; r <= row + radius && r < dc.H; ++r)
          for (int c = col - radius; c <= col + radius && c < dc.W; ++c) {
            const int q = r * dc.W + c;
            if (!M.exists[q]) continue;
            const double qr = M.rho[q];
            if (!(qr > -1e-6)) continue;
            const double diff = fabs(rho - qr);
            if (diff < sig || diff < 2.0 * sqrt(M.var[q])) mean += qr * (1.0 / M.var[q]) / tot;
          }
      } else mean = rho_post;
      isSet = true;
    }
  }
  M.rho_tmp[pix] = isSet ? mean : -1.0;
}
// Warp-cooperative form over the active list (one fold since the reset): one warp per listed pixel, lanes = 32 consecutive
// neighbours of the (2r+1)^2 window in raster order.  Validity / closeness tests run lane-parallel; the order-dependent
// Student-t merge of the close neighbours (DepthRegularization.cpp:63-86: sequential, non-associative in floating point) is
// replayed in raster order by broadcasting one close neighbour at a time.  Same arithmetic, same order as the thread form
// above; what changes is the latency: 121 (r = 5) ... 1681 (r = 20) dependent neighbour visits become 4 ... 53 chunk loads.
__global__ void __launch_bounds__(256, 3) map_regularize_warp_kernel(DevConsts dc, MapSoA M, int radius, int min_nb, int min_close,
                                                                  const int32_t* __restrict__ active, const unsigned long long* __restrict__ scal) {
  const unsigned FULLM = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int nwarps = gridDim.x * wpb;
  const int n_active = (int)scal[3];
  const int side = 2 * radius + 1, nn = side * side;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < n_active; t += nwarps) {
    const int pix = active[t];
    if (!M.exists[pix]) continue;
    const double rho = M.rho[pix];
    if (!(rho > -1e-6)) { if (lane == 0) M.rho_tmp[pix] = rho; continue; }
    const int row = pix / dc.W, col = pix - row * dc.W;
    bool isSet = false;
    double mean = 0;
    if (row >= radius && col >= radius) {   // SmartGrid::getNeighbourhood's int/size_t loop never runs otherwise (SmartGrid.h:373-375)
      const double sig = 2.0 * sqrt(M.var[pix]);
      int nb = 0, nclose = 0;
      double nu_post = 0, rho_post = 0, s2_post = 0, tot = 0;
      for (int k0 = 0; k0 < nn; k0 += 32) {
        const int k = k0 + lane;
        bool valid = false, close = false;
        double qr = 0, qv = 0;
        int q = 0;
        if (k < nn) {
          const int dr = k / side, dcc = k - dr * side;
          const int r = row - radius + dr, c = col - radius + dcc;
          if (r < dc.H && c < dc.W) {
            q = r * dc.W + c;
            if (M.exists[q]) {
              qr = M.rho[q];
              if (qr > -1e-6) {
                valid = true;
                qv = M.var[q];
                const double diff = fabs(rho - qr);
                close = diff < sig || diff < 2.0 * sqrt(qv);
              }
            }
          }
        }
        nb += __popc(__ballot_sync(FULLM, valid));
        unsigned cm = __ballot_sync(FULLM, close);
        double q_nu = 0, q_s2 = 0;
        if (close && dc.lsnorm != ESVO_LSNORM_L2) { q_nu = M.nu[q]; q_s2 = M.s2[q]; }
        while (cm) {
          const int src = __ffs(cm) - 1;
          cm &= cm - 1;
          const double rho_obs = __shfl_sync(FULLM, qr, src);
          if (dc.lsnorm == ESVO_LSNORM_L2) tot += 1.0 / __shfl_sync(FULLM, qv, src);
          else {
            const double nu_obs = __shfl_sync(FULLM, q_nu, src), s2_obs = __shfl_sync(FULLM, q_s2, src);
            if (nclose == 0) { nu_post = nu_obs; rho_post = rho_obs; s2_post = s2_obs; }
            else {
              const double nu_prior = nu_post, rho_prior = rho_post, s2_prior = s2_post;
              nu_post = fmin(nu_prior, nu_obs);
              rho_post = (s2_obs * rho_prior + s2_prior * rho_obs) / (s2_obs + s2_prior);
              const double d = rho_prior - rho_obs;
              s2_post = (nu_post + (d * d) / (s2_prior + s2_obs)) / (nu_post + 1) * (s2_prior * s2_obs) / (s2_prior + s2_obs);
            }
          }
          nclose++;
        }
      }
      if (nb > min_nb && nclose > min_close) {
        if (dc.lsnorm == ESVO_LSNORM_L2) {
          for (int k0 = 0; k0 < nn; k0 += 32) {      // second sweep: mean += qr * (1/var) / tot in raster order
            const int k = k0 + lane;
            bool close = false; double qr = 0, qv = 1;
            if (k < nn) {
              const int dr = k / side, dcc = k - dr * side;
              const int r = row - radius + dr, c = col - radius + dcc;
              if (r < dc.H && c < dc.W) {
                const int q = r * dc.W + c;
                if (M.exists[q]) { qr = M.rho[q]; if (qr > -1e-6) { qv = M.var[q]; const double diff = fabs(rho - qr); close = diff < sig || diff < 2.0 * sqrt(qv); } }
              }
            }
            unsigned cm = __ballot_sync(FULLM, close);
            while (cm) {
              const int src = __ffs(cm) - 1; cm &= cm - 1;
              mean += __shfl_sync(FULLM, qr, src) * (1.0 / __shfl_sync(FULLM, qv, src)) / tot;
            }
          }
        } else mean = rho_post;
        isSet = true;
      }
    }
    if (lane == 0) M.rho_tmp[pix] = isSet ? mean : -1.0;
  }
}
__global__ void map_regularize_commit_kernel(int npix, MapSoA M) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix < npix && M.exists[pix]) M.rho[pix] = M.rho_tmp[pix];
}
// list form of commit (+ the element count of map_count_kernel): scal[2] += number of existing pixels
__global__ void map_commit_count_list_kernel(MapSoA M, int commit, const int32_t* __restrict__ active, unsigned long long* scal) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  int e = 0;
  if ((unsigned long long)t < scal[3]) {
    const int pix = active[t];
    e = M.exists[pix] ? 1 : 0;
    if (e && commit) M.rho[pix] = M.rho_tmp[pix];
  }
  const int s = warp_sum_i(e);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(&scal[2], (unsigned long long)s);
}
// ---- ordered hand-off without sorting (one fold since the reset): the element list order is the order of the creating
// contribution ids; fuse_fold_kernel left one bit per surviving creator.  (1) exclusive popcount prefix per bitmap word
// (single block, a few thousand words), (2) every existing active pixel writes its element at position
// rank = prefix[word] + popc(bits below) -- straight into the (pinned, device-mapped) destination.
__device__ int block_excl_scan(int v, int* s_warp, int& total);
__global__ void __launch_bounds__(1024) map_cbits_prefix_kernel(const uint32_t* __restrict__ bits, uint32_t* __restrict__ prefix, int nwords,
                                                                unsigned long long* scal, unsigned long long* h_scal8,
                                                                const uint64_t* __restrict__ d_counters, uint64_t* h_counters) {
  __shared__ int s_warp[33];
  const int per = (nwords + 1023) / 1024;
  const int w0 = threadIdx.x * per, w1 = min(nwords, w0 + per);
  int cnt = 0;
  for (int w = w0; w < w1; ++w) cnt += __popc(bits[w]);
  int total;
  int run = block_excl_scan(cnt, s_warp, total);
  for (int w = w0; w < w1; ++w) { prefix[w] = (uint32_t)run; run += __popc(bits[w]); }
  if (threadIdx.x == 0) {
    scal[1] = (unsigned long long)total;
    if (h_scal8) { h_scal8[1] = (unsigned long long)total; h_scal8[4] = scal[0]; h_scal8[6] = scal[2]; }   // count, n_fusions, map size
  }
  if (h_counters && threadIdx.x < kCounters) h_counters[threadIdx.x] = d_counters[threadIdx.x];
}
__global__ void map_gather_list_kernel(MapSoA M, Pose16 Twf, const int32_t* __restrict__ active, const unsigned long long* __restrict__ scal,
                                       const uint32_t* __restrict__ bits, const uint32_t* __restrict__ prefix, esvo_depth_point* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = (unsigned long long)t < scal[3];
  const int pix = in ? active[t] : 0;
  const bool ex = in && M.exists[pix];
  unsigned rank = 0;
  if (ex) { const unsigned long long c = M.first_key[pix]; rank = prefix[c >> 5] + __popc(bits[c >> 5] & ((1u << (c & 31)) - 1u)); }
  // warp-cooperative element writes (28 x 8-byte words each): lane w moves word w of one element at a time
  constexpr int WORDS = sizeof(esvo_depth_point) / 8;
  const unsigned lane = threadIdx.x & 31u;
  const unsigned exmask = __ballot_sync(0xffffffffu, ex);
  for (unsigned e = 0; e < 32; ++e) {
    if (!((exmask >> e) & 1u)) continue;
    const unsigned r = __shfl_sync(0xffffffffu, rank, e);
    const int q = __shfl_sync(0xffffffffu, pix, e);
    if (lane < WORDS) {
      unsigned long long v;
      switch (lane) {
        case 0: { const unsigned long long lo = (unsigned)M.row[q], hi = (unsigned)M.col[q]; v = lo | (hi << 32); break; }
        case 1: v = __double_as_longlong(M.x0[q]); break;
        case 2: v = __double_as_longlong(M.x1[q]); break;
        case 3: v = __double_as_longlong(M.rho[q]); break;
        case 4: v = __double_as_longlong(M.s2[q]); break;
        case 5: v = __double_as_longlong(M.nu[q]); break;
        case 6: v = __double_as_longlong(M.var[q]); break;
        case 7: v = __double_as_longlong(M.res[q]); break;
        case 8: v = (unsigned long long)M.age[q]; break;
        case 9: v = __double_as_longlong(M.pc0[q]); break;
        case 10: v = __double_as_longlong(M.pc1[q]); break;
        case 11: v = __double_as_longlong(M.pc2[q]); break;
        default: v = __double_as_longlong(Twf.m[lane - 12]); break;
      }
      reinterpret_cast<unsigned long long*>(out + r)[lane] = v;
    }
  }
}

// ---- download: compact existing pixels (unordered) with their creation keys ----
__global__ void map_gather_kernel(DevConsts dc, MapSoA M, Pose16 TwfP, esvo_depth_point* out,
                                  unsigned long long* keys, unsigned long long* scal) {
  const double* Twf = TwfP.m;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= dc.W * dc.H || !M.exists[pix]) return;
  const unsigned long long pos = atomicAdd(&scal[1], 1ULL);
  esvo_depth_point d;
  d.row = M.row[pix]; d.col = M.col[pix]; d.x[0] = M.x0[pix]; d.x[1] = M.x1[pix]; d.inv_depth = M.rho[pix];
  d.scale2 = M.s2[pix]; d.nu = M.nu[pix]; d.variance = M.var[pix]; d.residual = M.res[pix]; d.age = M.age[pix];
  d.p_cam[0] = M.pc0[pix]; d.p_cam[1] = M.pc1[pix]; d.p_cam[2] = M.pc2[pix];
#pragma unroll
  for (int q = 0; q < 16; ++q) d.T_world_cam[q] = Twf[q];
  out[pos] = d;
  keys[pos] = M.first_key[pix];
}
// ---- ordered hand-off: rank every gathered element by its creation key and write it, in SmartGrid list order,
// straight into (pinned, device-mapped) host memory.  rank_i = #{ j : key_j < key_i } by brute force over shared
// memory tiles: n^2 compares, cheap for the usual few thousand map points.
__global__ void __launch_bounds__(256) map_rank_permute_kernel(const esvo_depth_point* __restrict__ in,
                                                               const unsigned long long* __restrict__ keys,
                                                               const unsigned long long* __restrict__ scal,
                                                               esvo_depth_point* __restrict__ out) {
  __shared__ unsigned long long tile[1024];
  const unsigned n = (unsigned)scal[1];
  if (blockIdx.x * 256u >= n) return;
  const unsigned i = blockIdx.x * 256u + threadIdx.x;
  const unsigned long long my = i < n ? keys[i] : ~0ULL;
  unsigned rank = 0;
  for (unsigned base = 0; base < n; base += 1024) {
    __syncthreads();
    for (unsigned k = threadIdx.x; k < 1024; k += 256) tile[k] = base + k < n ? keys[base + k] : ~0ULL;
    __syncthreads();
    const unsigned m = min(1024u, n - base);
#pragma unroll 8
    for (unsigned k = 0; k < m; ++k) rank += tile[k] < my ? 1u : 0u;
  }
  // warp-cooperative copy: WORDS (= 28) lanes move the 8-byte words of one element at a time (coalesced PCIe writes)
  constexpr int WORDS = sizeof(esvo_depth_point) / 8;
  static_assert(sizeof(esvo_depth_point) % 8 == 0 && WORDS <= 32, "element copy assumes <= 32 8-byte words");
  const unsigned lane = threadIdx.x & 31u, wbase = i - lane;
  for (unsigned e = 0; e < 32; ++e) {
    const unsigned r = __shfl_sync(0xffffffffu, rank, e);
    if (wbase + e < n && lane < WORDS)
      reinterpret_cast<unsigned long long*>(out + r)[lane] = reinterpret_cast<const unsigned long long*>(in + wbase + e)[lane];
  }
}

// ---- InitializationAtTime downstream of SGM (esvo_Mapping.cpp:446-480) + createEdgeMask (:1000-1044, undistorted
// events, radius 0): one DepthPoint per event whose rectified pixel carries a valid, in-range disparity, kept in
// event order (single-block ordered compaction, a few thousand events once at start-up).
__device__ int block_excl_scan(int v, int* s_warp, int& total);
// PerspectiveCamera::cam2World as the reference writes it (CameraSystem.cpp:120-139): invert [P; 0 0 0 z] and apply
// it to (x, y, 1, 1).  The SGM points sit on exact integer pixels and are re-projected through T_frame_obs ~ I right
// away, so floor(x) of the re-projection is decided by the last bit of p_cam: here (and only here) the device follows
// the cofactor expansion operation by operation instead of using the closed form.
__device__ bool inverse4_dev(const double* m, double* inv) {
  double t[16];
  t[0] = m[5]*m[10]*m[15] - m[5]*m[11]*m[14] - m[9]*m[6]*m[15] + m[9]*m[7]*m[14] + m[13]*m[6]*m[11] - m[13]*m[7]*m[10];
  t[4] = -m[4]*m[10]*m[15] + m[4]*m[11]*m[14] + m[8]*m[6]*m[15] - m[8]*m[7]*m[14] - m[12]*m[6]*m[11] + m[12]*m[7]*m[10];
  t[8] = m[4]*m[9]*m[15] - m[4]*m[11]*m[13] - m[8]*m[5]*m[15] + m[8]*m[7]*m[13] + m[12]*m[5]*m[11] - m[12]*m[7]*m[9];
  t[12] = -m[4]*m[9]*m[14] + m[4]*m[10]*m[13] + m[8]*m[5]*m[14] - m[8]*m[6]*m[13] - m[12]*m[5]*m[10] + m[12]*m[6]*m[9];
  t[1] = -m[1]*m[10]*m[15] + m[1]*m[11]*m[14] + m[9]*m[2]*m[15] - m[9]*m[3]*m[14] - m[13]*m[2]*m[11] + m[13]*m[3]*m[10];
  t[5] = m[0]*m[10]*m[15] - m[0]*m[11]*m[14] - m[8]*m[2]*m[15] + m[8]*m[3]*m[14] + m[12]*m[2]*m[11] - m[12]*m[3]*m[10];
  t[9] = -m[0]*m[9]*m[15] + m[0]*m[11]*m[13] + m[8]*m[1]*m[15] - m[8]*m[3]*m[13] - m[12]*m[1]*m[11] + m[12]*m[3]*m[9];
  t[13] = m[0]*m[9]*m[14] - m[0]*m[10]*m[13] - m[8]*m[1]*m[14] + m[8]*m[2]*m[13] + m[12]*m[1]*m[10] - m[12]*m[2]*m[9];
  t[2] = m[1]*m[6]*m[15] - m[1]*m[7]*m[14] - m[5]*m[2]*m[15] + m[5]*m[3]*m[14] + m[13]*m[2]*m[7] - m[13]*m[3]*m[6];
  t[6] = -m[0]*m[6]*m[15] + m[0]*m[7]*m[14] + m[4]*m[2]*m[15] - m[4]*m[3]*m[14] - m[12]*m[2]*m[7] + m[12]*m[3]*m[6];
  t[10] = m[0]*m[5]*m[15] - m[0]*m[7]*m[13] - m[4]*m[1]*m[15] + m[4]*m[3]*m[13] + m[12]*m[1]*m[7] - m[12]*m[3]*m[5];
  t[14] = -m[0]*m[5]*m[14] + m[0]*m[6]*m[13] + m[4]*m[1]*m[14] - m[4]*m[2]*m[13] - m[12]*m[1]*m[6] + m[12]*m[2]*m[5];
  t[3] = -m[1]*m[6]*m[11] + m[1]*m[7]*m[10] + m[5]*m[2]*m[11] - m[5]*m[3]*m[10] - m[9]*m[2]*m[7] + m[9]*m[3]*m[6];
  t[7] = m[0]*m[6]*m[11] - m[0]*m[7]*m[10] - m[4]*m[2]*m[11] + m[4]*m[3]*m[10] + m[8]*m[2]*m[7] - m[8]*m[3]*m[6];
  t[11] = -m[0]*m[5]*m[11] + m[0]*m[7]*m[9] + m[4]*m[1]*m[11] - m[4]*m[3]*m[9] - m[8]*m[1]*m[7] + m[8]*m[3]*m[5];
  t[15] = m[0]*m[5]*m[10] - m[0]*m[6]*m[9] - m[4]*m[1]*m[10] + m[4]*m[2]*m[9] + m[8]*m[1]*m[6] - m[8]*m[2]*m[5];
  double det = m[0]*t[0] + m[1]*t[4] + m[2]*t[8] + m[3]*t[12];
  if (det == 0) return false;
  det = 1.0 / det;
  for (int i = 0; i < 16; ++i) inv[i] = t[i] * det;
  return true;
}
__device__ void cam2world_general(const DevConsts& dc, double x, double y, double rho, double& p0, double& p1, double& p2) {
  const double z = 1.0 / rho;
  double Pt[16], Pi[16];
#pragma unroll
  for (int q = 0; q < 12; ++q) Pt[q] = dc.Pl[q];
  Pt[12] = 0; Pt[13] = 0; Pt[14] = 0; Pt[15] = z;
  inverse4_dev(Pt, Pi);
  const double xs[4] = {x, y, 1, 1};
  double ps[4];
  for (int i = 0; i < 4; ++i) {
    double s = 0;
    for (int k = 0; k < 4; ++k) s += (z * Pi[i * 4 + k]) * xs[k];
    ps[i] = s;
  }
  p0 = ps[0] / ps[3]; p1 = ps[1] / ps[3]; p2 = ps[2] / ps[3];
}
__global__ void __launch_bounds__(1024) sgm_points_kernel(DevConsts dc, const int16_t* __restrict__ disp16,
                                                          const uint16_t* __restrict__ ex, const uint16_t* __restrict__ ey, int n,
                                                          const double* __restrict__ lut, Pose16 TwcP,
                                                          double rho_min, double rho_max, long long age0, esvo_depth_point* out,
                                                          unsigned long long* out_cnt) {
  const double* T_world_cam = TwcP.m;
  __shared__ int s_warp[33];
  int running = 0;
  for (int k0 = 0; k0 < n; k0 += blockDim.x) {
    const int i = k0 + threadIdx.x;
    int f = 0, xc = 0, yc = 0;
    double rho = 0;
    if (i < n && ex[i] < dc.W && ey[i] < dc.H) {
      const size_t li = (size_t)ey[i] * dc.W + ex[i];
      const double cx = lut[2 * li], cy = lut[2 * li + 1];
      // floor()->int of a NaN / huge coordinate is UB in the reference; such events cannot be inside the image
      if (cx > -1e9 && cx < 1e9 && cy > -1e9 && cy < 1e9) {
        xc = (int)floor(cx); yc = (int)floor(cy);
        if (xc >= 0 && xc < dc.W && yc >= 0 && yc < dc.H) {
          const double disp = disp16[(size_t)yc * dc.W + xc] / 16.0;
          rho = disp / (dc.Pl[0] * dc.baseline);
          f = (!(disp < 0) && !(rho < rho_min || rho > rho_max)) ? 1 : 0;
        }
      }
    }
    int total;
    const int pos = running + block_excl_scan(f, s_warp, total);
    if (f) {
      esvo_depth_point* o = out + pos;
      o->row = xc; o->col = yc;                          // DepthPoint dp(x, y): the reference passes (x, y) as (row, col)
      o->x[0] = xc * 1.0; o->x[1] = yc * 1.0;
      double p0, p1, p2;
      cam2world_general(dc, xc * 1.0, yc * 1.0, rho, p0, p1, p2);
      o->p_cam[0] = p0; o->p_cam[1] = p1; o->p_cam[2] = p2;
      o->inv_depth = rho;
      { const double v = 0.001 * 0.001; o->variance = v < 1e-6 ? 1e-6 : v; }   // pow(0.001, 2), then boundVariance
      o->scale2 = 0; o->nu = 0;                          // never initialised by the reference for these points
      o->residual = 0.0; o->age = age0;
      for (int q = 0; q < 16; ++q) o->T_world_cam[q] = T_world_cam[q];
    }
    running += total;
  }
  if (threadIdx.x == 0) *out_cnt = (unsigned long long)running;
}
// T_world_cam = pose of the current map (host copy kept by fuse_reset_map), passed by value
int sgm_points(Ctx* c, const int16_t* d_disp, const uint16_t* d_ex, const uint16_t* d_ey, size_t n, esvo_depth_point* out,
               unsigned long long* out_cnt) {
  Pose16 Twc; std::memcpy(Twc.m, c->slot().map->T_world_frame, 128);
  sgm_points_kernel<<<1, 1024, 0, c->stream>>>(c->dc, d_disp, d_ex, d_ey, (int)n, c->d_lut, Twc, c->prm.invdepth_min_range,
                                               c->prm.invdepth_max_range, (long long)c->prm.age_vis_threshold, out, out_cnt);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

__global__ void fill_i32_kernel(int32_t* p, size_t n, int32_t v) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// --------------------------------------------------------------------------------------------
static int prop_reserve(Ctx* c, MapState* ms, size_t need) {
  if (need <= ms->prop_cap) return ESVO_OK;
  if (ms->staged) { c->set_error("internal: staging buffer grown while points are staged"); return ESVO_ERR_STATE; }
  size_t cap = std::max<size_t>(need, 65536);
  PropSoA& P = ms->p;
  void* olds[] = {P.hot, P.ok, P.rho, P.s2, P.nu, P.var, P.res, P.x0, P.x1, P.pc0, P.pc1, P.pc2, P.age, P.row, P.col, ms->next,
                  ms->cbits, ms->cprefix, ms->sort_pool};
  for (void* p : olds) if (p) cudaFree(p);
  ESVO_CUDA_TRY(c, dmalloc(&P.ok, cap)); ESVO_CUDA_TRY(c, dmalloc(&P.hot, cap));
  double** ds[] = {&P.rho, &P.s2, &P.nu, &P.var, &P.res, &P.x0, &P.x1, &P.pc0, &P.pc1, &P.pc2};
  for (double** d : ds) ESVO_CUDA_TRY(c, dmalloc(d, cap));
  ESVO_CUDA_TRY(c, dmalloc(&P.age, cap)); ESVO_CUDA_TRY(c, dmalloc(&P.row, cap)); ESVO_CUDA_TRY(c, dmalloc(&P.col, cap));
  ESVO_CUDA_TRY(c, dmalloc(&ms->next, cap * 9)); ESVO_CUDA_TRY(c, dmalloc(&ms->sort_pool, cap * 9));
  ms->cbits_words = (cap * 9 + 31) / 32;
  ESVO_CUDA_TRY(c, dmalloc(&ms->cbits, ms->cbits_words)); ESVO_CUDA_TRY(c, dmalloc(&ms->cprefix, ms->cbits_words));
  ms->prop_cap = cap;
  return ESVO_OK;
}

int fuse_alloc(Ctx* c, MapState** out) {
  MapState* ms = new MapState();
  *out = ms;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  MapSoA& M = ms->m;
  std::memset(&M, 0, sizeof(M)); std::memset(&ms->p, 0, sizeof(ms->p));
  ESVO_CUDA_TRY(c, dmalloc(&M.exists, npix));
  double** ds[] = {&M.rho, &M.s2, &M.nu, &M.var, &M.res, &M.x0, &M.x1, &M.pc0, &M.pc1, &M.pc2, &M.rho_tmp};
  for (double** d : ds) ESVO_CUDA_TRY(c, dmalloc(d, npix));
  ESVO_CUDA_TRY(c, dmalloc(&M.age, npix)); ESVO_CUDA_TRY(c, dmalloc(&M.row, npix)); ESVO_CUDA_TRY(c, dmalloc(&M.col, npix));
  ESVO_CUDA_TRY(c, dmalloc(&M.first_key, npix));
  ESVO_CUDA_TRY(c, dmalloc(&ms->head, npix));
  ESVO_CUDA_TRY(c, dmalloc(&ms->active, npix));
  ESVO_CUDA_TRY(c, dmalloc(&ms->pcnt, npix)); ESVO_CUDA_TRY(c, dmalloc(&ms->active_sorted, npix));
  ESVO_CUDA_TRY(c, cudaMemset(ms->pcnt, 0, npix * 4));       // invariant: every fold zeroes the counts it consumed
  ESVO_CUDA_TRY(c, dmalloc(&ms->d_dl, npix)); ESVO_CUDA_TRY(c, dmalloc(&ms->d_dl_keys, npix));
  ESVO_CUDA_TRY(c, dmalloc(&ms->d_scal, 8));
  ESVO_CUDA_TRY(c, cudaMallocHost((void**)&ms->h_scal, 4 * 8));
  ESVO_CUDA_TRY(c, cudaMemset(M.exists, 0, npix));
  ESVO_CUDA_TRY(c, cudaMemset(ms->head, 0xff, npix * 4));   // invariant: every fold leaves the heads it consumed at -1
  ESVO_CUDA_TRY(c, cudaMemset(ms->d_scal, 0, 8 * 8));
  for (int i = 0; i < 16; ++i) ms->T_world_frame[i] = ms->T_frame_world[i] = (i % 5 == 0) ? 1.0 : 0.0;
  ms->list_valid = true; ms->folds = 0;
  return prop_reserve(c, ms, 65536);
}
void fuse_free(MapState* ms) {
  if (!ms) return;
  MapSoA& M = ms->m; PropSoA& P = ms->p;
  void* ps[] = {M.exists, M.rho, M.s2, M.nu, M.var, M.res, M.x0, M.x1, M.pc0, M.pc1, M.pc2, M.rho_tmp, M.age, M.row, M.col,
                M.first_key, P.hot, P.ok, P.rho, P.s2, P.nu, P.var, P.res, P.x0, P.x1, P.pc0, P.pc1, P.pc2, P.age, P.row, P.col,
                ms->head, ms->next, ms->active, ms->pcnt, ms->active_sorted, ms->cbits, ms->cprefix, ms->sort_pool, ms->d_dl, ms->d_dl_keys, ms->d_scal};
  for (void* p : ps) if (p) cudaFree(p);
  if (ms->h_scal) cudaFreeHost(ms->h_scal);
  delete ms;
}

// New empty DepthFrame at pose T (esvo_Mapping.cpp:268-272).  Two enqueued operations: clear the existence plane and the
// map scalars {n_fusions, download count, map size, active pixels}.  The frame pose travels to the kernels by value.
int fuse_reset_map(Ctx* c, const double T[16]) {
  MapState* ms = c->slot().map;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  ESVO_CUDA_TRY(c, cudaMemsetAsync(ms->m.exists, 0, npix, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(ms->d_scal, 0, 64, c->stream));
  std::memcpy(ms->T_world_frame, T, 128);
  rigid_inverse(T, ms->T_frame_world);
  ms->seq_base = 0; ms->staged = 0;
  ms->list_valid = true; ms->folds = 0; ms->cleaned = false;
  return ESVO_OK;
}

// First staging call of a round that does not follow a reset: restart the active list (it then covers this round's pixels
// only, which is all the fold needs; kernels that need EVERY existing pixel fall back to their full-image form).
static int fuse_begin_round(Ctx* c) {
  MapState* ms = c->slot().map;
  if (ms->staged == 0 && ms->folds > 0) {
    ESVO_CUDA_TRY(c, cudaMemsetAsync(ms->d_scal + 3, 0, 24, c->stream));   // active count, (spare), sort-pool cursor
    ms->list_valid = false;
  }
  return ESVO_OK;
}

// Stage one vector of DepthPoints (device array).  n_cap bounds the count when it lives on the device.
// naive != 0: naive_propagate_one_point (:290-327) -- the Gaussian propagation whatever LSnorm is.
int fuse_points(Ctx* c, const esvo_depth_point* d_pts, size_t n_cap, const uint64_t* d_n, int radius, int naive) {
  MapState* ms = c->slot().map;
  if (n_cap == 0) return ESVO_OK;
  if (ms->staged + n_cap > ms->prop_cap) {
    if (ms->staged) { c->set_error("fusion staging capacity exceeded"); return ESVO_ERR_CAPACITY; }
    int rc = prop_reserve(c, ms, n_cap);
    if (rc) return rc;
  }
  int rc = fuse_begin_round(c);
  if (rc) return rc;
  const int B = 64;
  FrameSet fs;
  fs.nframes = 1; fs.pts[0] = d_pts; fs.cnt[0] = (const unsigned long long*)d_n; fs.cap[0] = (int)n_cap; fs.off[0] = 0; fs.off[1] = (int)n_cap;
  DevConsts dcs = c->dc;
  if (naive) dcs.lsnorm = ESVO_LSNORM_L2;
  Pose16 Tfw; std::memcpy(Tfw.m, ms->T_frame_world, 128);
  fuse_stage_kernel<<<div_up((int)n_cap, B), B, 0, c->stream>>>(dcs, fs, Tfw, radius, (int)ms->staged, ms->p, ms->head, ms->next,
                                                                ms->active, ms->pcnt, ms->d_scal);
  c->launches += 1;
  ms->staged += n_cap;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

// Stage a whole window (vectors given newest first) with as few launches as possible.
int fuse_window(Ctx* c, const Ctx::WinFrame* frames, int nframes, int radius) {
  MapState* ms = c->slot().map;
  const int B = 64;
  int rc = fuse_begin_round(c);
  if (rc) return rc;
  Pose16 Tfw; std::memcpy(Tfw.m, ms->T_frame_world, 128);
  for (int f0 = 0; f0 < nframes; f0 += FS_MAX) {
    FrameSet fs;
    fs.nframes = std::min(FS_MAX, nframes - f0);
    fs.off[0] = 0;
    for (int f = 0; f < fs.nframes; ++f) {
      fs.pts[f] = frames[f0 + f].pts; fs.cnt[f] = frames[f0 + f].cnt; fs.cap[f] = (int)frames[f0 + f].cap;
      fs.off[f + 1] = fs.off[f] + fs.cap[f];
    }
    const int tot = fs.off[fs.nframes];
    if (tot == 0) continue;
    if (ms->staged + (size_t)tot > ms->prop_cap) { c->set_error("fusion staging capacity exceeded"); return ESVO_ERR_CAPACITY; }
    fuse_stage_kernel<<<div_up(tot, B), B, 0, c->stream>>>(c->dc, fs, Tfw, radius, (int)ms->staged, ms->p, ms->head, ms->next, ms->active,
                                                           ms->pcnt, ms->d_scal);
    c->launches += 1;
    ms->staged += (size_t)tot;
  }
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

// Ordered per-pixel replay of everything staged since the last fold.  clean_* != null: SmartGrid::clean applied to the
// folded pixels on the way out (whole-frame path: the map was reset, so the folded pixels are all there is).
int fuse_finish(Ctx* c, bool naive, const double* clean4) {
  MapState* ms = c->slot().map;
  if (ms->staged == 0) return ESVO_OK;
  CleanArgs ca{0, 0, 0, 0, 0};
  if (clean4) { ca.enable = 1; ca.var_thr = clean4[0]; ca.age_thr = clean4[1]; ca.rmax = clean4[2]; ca.rmin = clean4[3]; }
  // creator bits feed the sort-free ordered hand-off; only meaningful for the first fold after a reset
  uint32_t* cbits = nullptr;
  if (ms->list_valid && ms->folds == 0) {
    ms->fold_words = (ms->staged * 9 + 31) / 32;
    ESVO_CUDA_TRY(c, cudaMemsetAsync(ms->cbits, 0, ms->fold_words * 4, c->stream));
    cbits = ms->cbits;
  }
  // Thread per active pixel: in the frame pipeline the fold's cost is warp-slot time next to the LM blocks, and a few hundred
  // dense warps beat thousands of one-pixel warps there, although a warp per pixel is faster alone.
  // At most one thread per image pixel can be active; the grid covers that bound, surplus blocks exit on the device count.
  const int npix = c->dc.W * c->dc.H, B = 32;
  const int bound = (int)std::min<size_t>((size_t)npix, ms->staged * 9);
  // pixels ordered by list length, longest first
  fold_order_kernel<<<1, 1024, 0, c->stream>>>(ms->active, ms->pcnt, ms->d_scal, ms->active_sorted);
  c->launches += 1;
  if (naive) fuse_fold_kernel<true><<<div_up(bound, B), B, 0, c->stream>>>(c->dc, ms->m, ms->p, ms->head, ms->next, ms->active_sorted, ms->pcnt, ms->seq_base, ms->d_scal, cbits, ca, ms->sort_pool);
  else fuse_fold_kernel<false><<<div_up(bound, B), B, 0, c->stream>>>(c->dc, ms->m, ms->p, ms->head, ms->next, ms->active_sorted, ms->pcnt, ms->seq_base, ms->d_scal, cbits, ca, ms->sort_pool);
  c->launches += 1;
  ms->seq_base += (unsigned long long)ms->staged * 9ULL;
  ms->staged = 0;
  ms->folds++;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}
static bool list_ok(const MapState* ms) { return ms->list_valid && ms->folds == 1; }

int map_clean(Ctx* c, double var_thr, double age_thr, double rmax, double rmin) {
  const int npix = c->dc.W * c->dc.H, B = 256;
  MapState* ms = c->slot().map;
  map_clean_kernel<<<div_up(npix, B), B, 0, c->stream>>>(npix, ms->m, var_thr, age_thr, rmax, rmin);
  c->launches += 1;
  ms->cleaned = true;
  return ESVO_OK;
}

// DepthRegularization::apply; count != 0 also leaves the number of map elements in d_scal[2] (zeroed by the reset).
int map_regularize(Ctx* c, bool count) {
  MapState* ms = c->slot().map;
  const int npix = c->dc.W * c->dc.H, B = 32;
  if (list_ok(ms)) {
    // persistent: one-warp blocks walk the active list, one warp per pixel.  One-warp blocks (4 K registers) slot into the
    // holes single LM blocks leave in a busy SM; bigger blocks wait for several neighbouring LM warps to retire.
    map_regularize_warp_kernel<<<c->num_sms * 16, 32, 0, c->stream>>>(c->dc, ms->m, c->prm.reg_radius, c->prm.reg_min_neighbours,
                                                                       c->prm.reg_min_close_neighbours, ms->active, ms->d_scal);
    if (count) map_commit_count_list_kernel<<<div_up(npix, 256), 256, 0, c->stream>>>(ms->m, 1, ms->active, ms->d_scal);
    else map_regularize_commit_kernel<<<div_up(npix, 256), 256, 0, c->stream>>>(npix, ms->m);
    c->launches += 2;
    return ESVO_OK;
  }
  map_regularize_kernel<<<div_up(npix, B), B, 0, c->stream>>>(c->dc, ms->m, c->prm.reg_radius, c->prm.reg_min_neighbours,
                                                              c->prm.reg_min_close_neighbours);
  map_regularize_commit_kernel<<<div_up(npix, 256), 256, 0, c->stream>>>(npix, ms->m);
  c->launches += 2;
  if (count) return map_count(c);
  return ESVO_OK;
}

// Enqueue (on c->stream) the compaction of the current map into caller-provided device buffers and the
// D2H of its scalars: h_scal8[1] = element count, h_scal8[4] = n_fusions, h_scal8[6] = map size.
// With h_sorted (pinned host memory, npix elements) the elements are also written there in creation order.
// h_counters (pinned, optional): receives a copy of the frame's kCounters device counters.
int map_gather_async(Ctx* c, esvo_depth_point* d_out, unsigned long long* d_keys, unsigned long long* d_scal4,
                     unsigned long long* h_scal8, esvo_depth_point* h_sorted, uint64_t* h_counters) {
  MapState* ms = c->slot().map;
  const int npix = c->dc.W * c->dc.H, B = 128;
  Pose16 Twf; std::memcpy(Twf.m, ms->T_world_frame, 128);
  if (h_sorted && list_ok(ms) && ms->fold_words && !ms->cleaned) {
    // sort-free: rank from the creator bitmap; the kernels write elements, scalars and counters straight into pinned memory
    map_cbits_prefix_kernel<<<1, 1024, 0, c->stream>>>(ms->cbits, ms->cprefix, (int)ms->fold_words, ms->d_scal, h_scal8, c->slot().d_counters, h_counters);
    map_gather_list_kernel<<<div_up(npix, B), B, 0, c->stream>>>(ms->m, Twf, ms->active, ms->d_scal, ms->cbits, ms->cprefix, h_sorted);
    c->launches += 2;
    ESVO_CUDA_TRY(c, cudaGetLastError());
    return ESVO_OK;
  }
  ESVO_CUDA_TRY(c, cudaMemsetAsync(d_scal4, 0, 32, c->stream));
  map_gather_kernel<<<div_up(npix, B), B, 0, c->stream>>>(c->dc, ms->m, Twf, d_out, d_keys, d_scal4);
  c->launches += 1;
  if (h_sorted) {
    map_rank_permute_kernel<<<div_up(npix, 256), 256, 0, c->stream>>>(d_out, d_keys, d_scal4, h_sorted);
    c->launches += 1;
  }
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h_scal8, d_scal4, 32, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h_scal8 + 4, ms->d_scal, 32, cudaMemcpyDeviceToHost, c->stream));
  if (h_counters) ESVO_CUDA_TRY(c, cudaMemcpyAsync(h_counters, c->slot().d_counters, kCounters * 8, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

// publishPointCloud's packing (esvo_Mapping.cpp:909-953, frontend::packPointCloud): p_world = R p_cam + t of every element,
// in element-list order, as pcl::PointXYZ.  The host code is built without FMA contraction, so each row is summed as
// ((T0 p0 + T1 p1) + T2 p2) + T3 with separately rounded products and one conversion to f32 at the end: the explicit
// _rn intrinsics keep that rounding whatever the compiler flags are.
__global__ void map_pack_cloud_kernel(const esvo_depth_point* __restrict__ e, int n, Pose16 Tp, float* __restrict__ xyz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* T = Tp.m;
  const double* p = e[i].p_cam;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * r], p[0]), __dmul_rn(T[4 * r + 1], p[1])), __dmul_rn(T[4 * r + 2], p[2])),
                               T[4 * r + 3]);
    xyz[3 * i + r] = __double2float_rn(s);
  }
}
// Element list in creation order (map_gather_async: creator-bit ranks after one fold, key ranks otherwise), then the pack.
// One host sync, for the count.
int map_publish(Ctx* c, const double T[16], size_t* n) {
  Ctx::Published& pb = c->pub;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  if (!pb.xyz) {
    ESVO_CUDA_TRY(c, dmalloc(&pb.xyz, 3 * npix)); ESVO_CUDA_TRY(c, dmalloc(&pb.sorted, npix)); ESVO_CUDA_TRY(c, dmalloc(&pb.d_scal, 4));
    ESVO_CUDA_TRY(c, cudaMallocHost((void**)&pb.h_scal, 8 * 8));
  }
  MapState* ms = c->slot().map;
  int rc = map_gather_async(c, ms->d_dl, ms->d_dl_keys, pb.d_scal, pb.h_scal, pb.sorted, nullptr);
  if (rc) return rc;
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  const int cnt = (int)pb.h_scal[1];
  Pose16 Tp; std::memcpy(Tp.m, T, 128);
  if (cnt) {
    map_pack_cloud_kernel<<<div_up(cnt, 128), 128, 0, c->stream>>>(pb.sorted, cnt, Tp, pb.xyz);
    c->launches += 1;
    ESVO_CUDA_TRY(c, cudaGetLastError());
  }
  *n = (size_t)cnt;
  return ESVO_OK;
}

int map_download(Ctx* c, esvo_depth_point* out, size_t* n) {
  MapState* ms = c->slot().map;
  const int npix = c->dc.W * c->dc.H, B = 128;
  Pose16 Twf; std::memcpy(Twf.m, ms->T_world_frame, 128);
  ESVO_CUDA_TRY(c, cudaMemsetAsync(ms->d_scal + 1, 0, 8, c->stream));
  map_gather_kernel<<<div_up(npix, B), B, 0, c->stream>>>(c->dc, ms->m, Twf, ms->d_dl, ms->d_dl_keys, ms->d_scal);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(ms->h_scal, ms->d_scal, 32, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  const size_t cnt = (size_t)ms->h_scal[1];
  if (cnt > *n) { *n = cnt; return ESVO_ERR_CAPACITY; }
  // Host marshalling: restore SmartGrid's list order (creation sequence) while copying out.
  std::vector<esvo_depth_point> tmp(cnt);
  std::vector<unsigned long long> keys(cnt);
  if (cnt) {
    ESVO_CUDA_TRY(c, cudaMemcpy(tmp.data(), ms->d_dl, cnt * sizeof(esvo_depth_point), cudaMemcpyDeviceToHost));
    ESVO_CUDA_TRY(c, cudaMemcpy(keys.data(), ms->d_dl_keys, cnt * 8, cudaMemcpyDeviceToHost));
  }
  std::vector<uint32_t> ord(cnt);
  for (size_t i = 0; i < cnt; ++i) ord[i] = (uint32_t)i;
  std::sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
  for (size_t i = 0; i < cnt; ++i) out[i] = tmp[ord[i]];
  *n = cnt;
  return ESVO_OK;
}

__global__ void map_count_kernel(int npix, MapSoA M, unsigned long long* scal) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int e = (pix < npix && M.exists[pix]) ? 1 : 0;
  const int s = warp_sum_i(e);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(&scal[2], (unsigned long long)s);
}
// counts existing map pixels into scal[2]
int map_count(Ctx* c) {
  MapState* ms = c->slot().map;
  if (list_ok(ms)) {   // scal[2] is still zero from the reset
    map_commit_count_list_kernel<<<div_up(c->dc.W * c->dc.H, 256), 256, 0, c->stream>>>(ms->m, 0, ms->active, ms->d_scal);
    c->launches += 1;
    return ESVO_OK;
  }
  const int npix = c->dc.W * c->dc.H, B = 256;
  ESVO_CUDA_TRY(c, cudaMemsetAsync(ms->d_scal + 2, 0, 8, c->stream));
  map_count_kernel<<<div_up(npix, B), B, 0, c->stream>>>(npix, ms->m, ms->d_scal);
  c->launches += 1;
  return ESVO_OK;
}
int fuse_zero_fusion_counter(Ctx* c) {
  ESVO_CUDA_TRY(c, cudaMemsetAsync(c->slot().map->d_scal, 0, 8, c->stream));
  return ESVO_OK;
}
// D2H of the map scalars: out[0] = n_fusions since the last zeroing, out[2] = map size (after map_count)
int fuse_fetch_scalars(Ctx* c, unsigned long long out[4]) {
  MapState* ms = c->slot().map;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(ms->h_scal, ms->d_scal, 32, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < 4; ++i) out[i] = ms->h_scal[i];
  return ESVO_OK;
}
int fuse_reserve(Ctx* c, size_t total_points) { return prop_reserve(c, c->slot().map, total_points); }

}  // namespace esvo
