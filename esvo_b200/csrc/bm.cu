// esvo_b200 product code -- event block matching along the epipolar line (sm_90a).
//
// Replaces esvo_core::core::EventBM::{match_an_event, epipolarSearching, zncc_cost, isValidPatch,
// match_all_HyperThread} (esvo_core/src/core/EventBM.cpp:80-333) and tools::normalizePatch
// (esvo_core/include/esvo_core/tools/utils.h:74-92).
//
// Design: one warp per event; the 32 lanes are 32 disparity candidates.  The time surfaces live in
// HBM as u8 (values are exact integers 0..255, so the reference's f64 copies carry no extra
// information); the left patch is staged once per event in shared memory, every lane accumulates
// the exact integer moments  S_r, S_rr, S_lr  of its candidate window and the ZNCC cost is then
// evaluated in f64 from those integers (mean = S/N is the same single rounding the reference
// performs; see DESIGN.md "BM cost" for the rounding discussion).  Algorithmic bytes per candidate:
// 105 px x 4 B = 420 B (SURVEY.md 8d, f32 TS convention).
#include <cuda.h>      // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint, libcuda is not linked)

#include "common.cuh"

namespace esvo {

constexpr int BM_WARPS = 1;   // one event per block (2.5 K registers): fits the hole a retiring LM block leaves (fuse.cu: fuse_finish)
constexpr int BM_MAXC = 192;  // max coarse candidates per event kept in shared memory

struct BmArgs {
  const uint16_t *ex, *ey;
  const int64_t* et;
  int n;
  const double* lut;
  const uint8_t* mask;
  const uint8_t *tl, *tr;
  const int64_t* pose_t;
  int n_poses;
  BmDense out;
  unsigned long long* counters;
};

__device__ __forceinline__ bool bm_valid_patch(int x, int y, int hx, int hy, int W, int H) {
  // EventBM::isValidPatch (EventBM.cpp:251-267)
  return !(x - hx < 1 || y - hy < 1 || x + hx >= W - 1 || y + hy >= H - 1);
}

__device__ __forceinline__ double bm_cost_from_moments(int N, int Sl, int Sll, int Sr, int Srr, int Slr) {
  // sigma = sqrt(sum((p-mean)^2)/N) + 1e-6 ; cost = 0.5*(1 - sum(l^ r^)/N)
  const double n = (double)N;
  double varl = (double)((long long)N * Sll - (long long)Sl * Sl) / (n * n);
  double varr = (double)((long long)N * Srr - (long long)Sr * Sr) / (n * n);
  double sl = sqrt(varl) + 1e-6, sr = sqrt(varr) + 1e-6;
  double cov = (double)((long long)N * Slr - (long long)Sl * Sr) / n;  // sum (l-ml)(r-mr)
  return 0.5 * (1.0 - (cov / (sl * sr)) / n);
}

__global__ void __launch_bounds__(BM_WARPS * 32) bm_kernel(DevConsts dc, BmArgs a) {
  __shared__ uint8_t s_left[BM_WARPS][kMaxPatch];
  __shared__ double s_cost[BM_WARPS][BM_MAXC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * BM_WARPS + warp;
  if (i >= a.n) return;
  const int W = dc.W, H = dc.H, wx = dc.wx, wy = dc.wy, N = wx * wy;
  const int hx = (wx - 1) / 2, hy = (wy - 1) / 2;
  if (lane == 0) a.out.flag[i] = 0;
  const int ex = a.ex[i], ey = a.ey[i];
  if (ex >= W || ey >= H) return;
  const size_t li = (size_t)ey * W + ex;
  const double xr0 = a.lut[2 * li], xr1 = a.lut[2 * li + 1];
  if (xr0 < 0 || xr0 > W - 1 || xr1 < 0 || xr1 > H - 1) return;            // :90-92
  if (a.mask[(size_t)((int)xr1) * W + (int)xr0] <= 125) return;             // :94
  const int x1x = (int)floor(xr0), x1y = (int)floor(xr1);
  if (!bm_valid_patch(x1x, x1y, hx, hy, W, H)) return;
  // left patch -> shared, moments + low-texture count (:101-109)
  int Sl = 0, Sll = 0, cnt0 = 0;
  for (int k = lane; k < N; k += 32) {
    int py = k / wx, px = k - py * wx;
    int v = a.tl[(size_t)(x1y - hy + py) * dc.pitch + (x1x - hx + px)];
    s_left[warp][k] = (uint8_t)v;
    Sl += v; Sll += v * v; cnt0 += (v < 1);
  }
  Sl = warp_sum_i(Sl); Sll = warp_sum_i(Sll); cnt0 = warp_sum_i(cnt0);
  __syncwarp();
  if ((double)cnt0 > 0.95 * (double)N) return;

  const int step = dc.step;
  const int ncand = (dc.dmax >= dc.dmin) ? (dc.dmax - dc.dmin) / step + 1 : 0;
  auto eval = [&](int disp, bool& valid) -> double {
    int x2x = dc.updown ? x1x : x1x - disp, x2y = dc.updown ? x1y - disp : x1y;
    valid = bm_valid_patch(x2x, x2y, hx, hy, W, H);
    if (!valid) return 1.0;
    const uint8_t* base = a.tr + (size_t)(x2y - hy) * dc.pitch + (x2x - hx);
    int Sr = 0, Srr = 0, Slr = 0;
    for (int py = 0; py < wy; ++py) {
      const uint8_t* row = base + (size_t)py * dc.pitch;
      const uint8_t* lrow = &s_left[warp][py * wx];
#pragma unroll 5
      for (int px = 0; px < wx; ++px) {
        int r = row[px], l = lrow[px];
        Sr += r; Srr += r * r; Slr += l * r;
      }
    }
    return bm_cost_from_moments(N, Sl, Sll, Sr, Srr, Slr);
  };

  // ---- coarse search (:119): lanes = candidates ----
  double best = 1.0; int bestDisp = -1; int nev = 0;
  for (int j = lane; j < ncand; j += 32) {
    bool valid; int disp = dc.dmin + j * step;
    double c = eval(disp, valid);
    nev += valid;
    if (j < BM_MAXC) s_cost[warp][j] = c;
    if (valid && c <= best) { best = c; bestDisp = disp; }   // later disparity wins ties (:198)
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ob = __shfl_xor_sync(0xffffffffu, best, o); int od = __shfl_xor_sync(0xffffffffu, bestDisp, o);
    if (od >= 0 && (bestDisp < 0 || ob < best || (ob == best && od > bestDisp))) { best = ob; bestDisp = od; }
  }
  nev = warp_sum_i(nev);
  __syncwarp();
  bool coarse_ok = false;
  if (bestDisp >= 0) {
    if (step > 1) {  // :204-215  both neighbours must exist in the cost map with cost < ZNCC_MAX
      int jb = (bestDisp - dc.dmin) / step;
      if (jb - 1 >= 0 && jb + 1 < ncand && jb + 1 < BM_MAXC)
        coarse_ok = s_cost[warp][jb - 1] < 1.0 && s_cost[warp][jb + 1] < 1.0 && best < dc.zncc_thr;
    } else coarse_ok = best < dc.zncc_thr;                                  // :217-221
  }
  if (!coarse_ok) { if (lane == 0) atomicAdd(&a.counters[5], (unsigned long long)nev); return; }
  // ---- fine search (:126-136): [bestDisp-(step-1), bestDisp+(step-1)], min_cost carried over ----
  int nev2 = 0;
  if (bestDisp >= step - 1) {
    const int f0 = bestDisp - (step - 1), nf = 2 * (step - 1) + 1;
    double fb = 2.0; int fd = -1;
    for (int j = lane; j < nf; j += 32) {
      bool valid; double c = eval(f0 + j, valid);
      nev2 += valid;
      if (valid && c <= (fd < 0 ? best : fb)) { fb = c; fd = f0 + j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      double ob = __shfl_xor_sync(0xffffffffu, fb, o); int od = __shfl_xor_sync(0xffffffffu, fd, o);
      if (od >= 0 && (fd < 0 || ob < fb || (ob == fb && od > fd))) { fb = ob; fd = od; }
    }
    nev2 = warp_sum_i(nev2);
    if (fd >= 0 && fb <= best) { best = fb; bestDisp = fd; }  // fine candidates come later in the sequence
  }
  if (lane == 0) atomicAdd(&a.counters[5], (unsigned long long)(nev + nev2));
  if (!(best < dc.zncc_thr)) return;   // fine-search success (:217-221) and accept test (:141)
  // StampTransformationMap_lower_bound (utils.h:64-69): first pose with toSec(stamp) >= toSec(t_event)
  if (lane == 0) {
    const double te = ns_to_sec_dev(a.et[i]);
    int lo = 0, hi = a.n_poses;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (ns_to_sec_dev(a.pose_t[mid]) < te) lo = mid + 1; else hi = mid; }
    if (lo == a.n_poses) return;                                            // :155-156
    a.out.disp[i] = bestDisp; a.out.pose_idx[i] = lo; a.out.cost[i] = best;
    a.out.xrect[2 * i] = xr0; a.out.xrect[2 * i + 1] = xr1;
    a.out.flag[i] = 1;
  }
}

// --------------------------------------------------------------------------------------------
// TMA form (the default since round 2; VERDICT r1 item 9): the right-image strip every candidate window of one event lies in --
// wy rows x (wx + dmax - dmin) bytes -- is fetched with ONE cp.async.bulk.tensor.2d (tensor map over the pitched u8
// surface, zero fill outside the image) into shared memory behind an mbarrier; the 32 lanes then read their candidate windows
// from shared memory instead of issuing per-lane LDG.E.U8 against L1.  Same arithmetic, same results as bm_kernel (horizontal
// search, step 1 only).
// --------------------------------------------------------------------------------------------
template <int BW>     // box width in bytes (multiple of 16)
__global__ void __launch_bounds__(32) bm_tma_kernel(DevConsts dc, BmArgs a, const __grid_constant__ CUtensorMap tmap_r) {
  __shared__ __align__(128) uint8_t s_strip[8 * BW];
  __shared__ uint8_t s_left[kMaxPatch];
  __shared__ __align__(8) unsigned long long s_bar;
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x;
  if (i >= a.n) return;
  const int W = dc.W, H = dc.H, wx = dc.wx, wy = dc.wy, N = wx * wy;
  const int hx = (wx - 1) / 2, hy = (wy - 1) / 2;
  if (lane == 0) a.out.flag[i] = 0;
  const int ex = a.ex[i], ey = a.ey[i];
  if (ex >= W || ey >= H) return;
  const size_t li = (size_t)ey * W + ex;
  const double xr0 = a.lut[2 * li], xr1 = a.lut[2 * li + 1];
  if (xr0 < 0 || xr0 > W - 1 || xr1 < 0 || xr1 > H - 1) return;
  if (a.mask[(size_t)((int)xr1) * W + (int)xr0] <= 125) return;
  const int x1x = (int)floor(xr0), x1y = (int)floor(xr1);
  if (!bm_valid_patch(x1x, x1y, hx, hy, W, H)) return;
  // issue the strip load first: it flies while the left patch is staged and tested
  // the inner coordinate of a TMA box load must be 16-byte aligned (an unaligned x raises "illegal instruction"): load from
  // the aligned column below and carry the offset
  const int x_want = x1x - dc.dmax - hx, y_lo = x1y - hy;
  const int x_lo = x_want & ~15, x_off = x_want - x_lo;
  const unsigned bar = (unsigned)__cvta_generic_to_shared(&s_bar), dst = (unsigned)__cvta_generic_to_shared(s_strip);
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((unsigned)(BW * wy)) : "memory");
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(&tmap_r)), "r"(bar), "r"(x_lo), "r"(y_lo) : "memory");
  }
  int Sl = 0, Sll = 0, cnt0 = 0;
  for (int k = lane; k < N; k += 32) {
    int py = k / wx, px = k - py * wx;
    int v = a.tl[(size_t)(x1y - hy + py) * dc.pitch + (x1x - hx + px)];
    s_left[k] = (uint8_t)v;
    Sl += v; Sll += v * v; cnt0 += (v < 1);
  }
  Sl = warp_sum_i(Sl); Sll = warp_sum_i(Sll); cnt0 = warp_sum_i(cnt0);
  __syncwarp();
  {  // every lane waits for the strip (phase 0); the block must not exit while the copy is in flight
    unsigned done = 0;
    while (!done) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.b32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar) : "memory");
  }
  if ((double)cnt0 > 0.95 * (double)N) return;
  const int ncand = (dc.dmax >= dc.dmin) ? (dc.dmax - dc.dmin) + 1 : 0;
  double best = 1.0; int bestDisp = -1; int nev = 0;
  for (int j = lane; j < ncand; j += 32) {
    const int disp = dc.dmin + j;
    const int x2x = x1x - disp;
    const bool valid = bm_valid_patch(x2x, x1y, hx, hy, W, H);
    double c = 1.0;
    if (valid) {
      const uint8_t* base = s_strip + x_off + (dc.dmax - disp);
      int Sr = 0, Srr = 0, Slr = 0;
      for (int py = 0; py < wy; ++py) {
        const uint8_t* row = base + py * BW;
        const uint8_t* lrow = &s_left[py * wx];
#pragma unroll 5
        for (int px = 0; px < wx; ++px) { int r = row[px], l = lrow[px]; Sr += r; Srr += r * r; Slr += l * r; }
      }
      c = bm_cost_from_moments(N, Sl, Sll, Sr, Srr, Slr);
    }
    nev += valid;
    if (valid && c <= best) { best = c; bestDisp = disp; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ob = __shfl_xor_sync(0xffffffffu, best, o); int od = __shfl_xor_sync(0xffffffffu, bestDisp, o);
    if (od >= 0 && (bestDisp < 0 || ob < best || (ob == best && od > bestDisp))) { best = ob; bestDisp = od; }
  }
  nev = warp_sum_i(nev);
  const bool coarse_ok = bestDisp >= 0 && best < dc.zncc_thr;
  if (!coarse_ok) { if (lane == 0) atomicAdd(&a.counters[5], (unsigned long long)nev); return; }
  // fine search of step 1 re-evaluates the best candidate once (EventBM.cpp:126-136): same cost, one more evaluation
  if (lane == 0) atomicAdd(&a.counters[5], (unsigned long long)(nev + 1));
  if (!(best < dc.zncc_thr)) return;
  if (lane == 0) {
    const double te = ns_to_sec_dev(a.et[i]);
    int lo = 0, hi = a.n_poses;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (ns_to_sec_dev(a.pose_t[mid]) < te) lo = mid + 1; else hi = mid; }
    if (lo == a.n_poses) return;
    a.out.disp[i] = bestDisp; a.out.pose_idx[i] = lo; a.out.cost[i] = best;
    a.out.xrect[2 * i] = xr0; a.out.xrect[2 * i + 1] = xr1;
    a.out.flag[i] = 1;
  }
}

typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
bool make_u8_tensor_map(CUtensorMap* tm, const uint8_t* img, int W, int H, int pitch, int boxw, int boxh) {
  static tmap_encode_fn enc = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) fn = nullptr;
    return (tmap_encode_fn)fn;
  }();
  if (!enc) return false;
  const cuuint64_t gdim[2] = {(cuuint64_t)W, (cuuint64_t)H};
  const cuuint64_t gstr[1] = {(cuuint64_t)pitch};
  const cuuint32_t box[2] = {(cuuint32_t)boxw, (cuuint32_t)boxh}, estr[2] = {1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)img, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// --------------------------------------------------------------------------------------------
// Ordered compaction.  The reference fans events out to NT threads with the interleave
// i = tid, tid+NT, ... and concatenates the per-thread result vectors (EventBM.cpp:295-315,
// DepthProblemSolver.cpp:65-90), so position(i) = #accepted in classes < i%NT + #accepted
// j<i with j%NT == i%NT.  Single block; the inputs are a few thousand flags.
// --------------------------------------------------------------------------------------------
__device__ int block_excl_scan(int v, int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nw ? s_warp[lane] : 0, wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
    s_warp[lane] = wi - w;            // exclusive per-warp offsets
    if (lane == 31) s_warp[32] = wi;  // grand total
  }
  __syncthreads();
  int res = s_warp[warp] + inc - v;
  total = s_warp[32];
  __syncthreads();
  return res;
}

// virtual position v in the thread-major order -> event index i
__device__ __forceinline__ int tm_index(int v, int n, int NT) {
  int c = 0, start = 0;
  for (; c < NT; ++c) {
    const int members = (n > c) ? (n - c + NT - 1) / NT : 0;
    if (v < start + members) break;
    start += members;
  }
  return c + (v - start) * NT;
}

// Multi-block ordered compaction without inter-block communication: block b owns the virtual positions [256 b, 256 b + 256)
// of the thread-major order; its base offset is the number of accepted events at EARLIER virtual positions, which the block
// simply counts itself (b x 256 flag reads, L2-resident -- a few thousand flags in total), followed by a block scan of its own
// 256 flags.  No look-back state, nothing to zero, every block independent.  The last block publishes the total.
constexpr int kOrdBlock = 256;
__global__ void __launch_bounds__(kOrdBlock) seeds_order_kernel(DevConsts dc, BmDense d, const uint16_t* __restrict__ ex,
                                                                const uint16_t* __restrict__ ey, const int64_t* __restrict__ et,
                                                                const double* __restrict__ poses, int n, esvo_seed* out,
                                                                unsigned long long* counters) {
  __shared__ int s_warp[33];
  __shared__ int s_base;
  const int NT = dc.NT;
  const int v0 = blockIdx.x * kOrdBlock;
  if (v0 >= n) return;
  int pre = 0;
  for (int v = threadIdx.x; v < v0; v += kOrdBlock) pre += d.flag[tm_index(v, n, NT)];
  int tot_pre;
  block_excl_scan(pre, s_warp, tot_pre);
  if (threadIdx.x == 0) s_base = tot_pre;
  const int v = v0 + threadIdx.x;
  const int i = v < n ? tm_index(v, n, NT) : 0;
  const int f = v < n ? d.flag[i] : 0;
  int total;
  const int local = block_excl_scan(f, s_warp, total);
  const int pos = s_base + local;
  if (f) {
    esvo_seed s;
    s.x_left_raw[0] = (double)ex[i]; s.x_left_raw[1] = (double)ey[i];
    const double xr0 = d.xrect[2 * i], xr1 = d.xrect[2 * i + 1];
    s.x_left[0] = xr0; s.x_left[1] = xr1;
    const int x1x = (int)floor(xr0), x1y = (int)floor(xr1), disp = d.disp[i];
    s.x_right[0] = (double)(dc.updown ? x1x : x1x - disp);
    s.x_right[1] = (double)(dc.updown ? x1y - disp : x1y);
    s.t_ns = et[i];
    const double* T = poses + 16 * (size_t)d.pose_idx[i];
#pragma unroll
    for (int q = 0; q < 16; ++q) s.T_world_virtual[q] = T[q];
    const double disparity = (double)disp;
    const double depth = dc.baseline * dc.Pl[0] / disparity;           // EventBM.cpp:152
    s.inv_depth = 1.0 / depth; s.cost = d.cost[i]; s.disp = disparity;
    out[pos] = s;
  }
  if (v0 + kOrdBlock >= n && threadIdx.x == 0) counters[1] = (unsigned long long)(s_base + total);
}

// --------------------------------------------------------------------------------------------
// host launchers
// --------------------------------------------------------------------------------------------
int bm_run(Ctx* c) {
  const SlotBufs& f = c->slot();
  if (f.n_ev == 0) return ESVO_OK;
  BmArgs a;
  a.ex = f.d_ex; a.ey = f.d_ey; a.et = f.d_et; a.n = (int)f.n_ev; a.lut = c->d_lut; a.mask = c->d_mask;
  a.tl = f.obs_ls; a.tr = f.obs_rs; a.pose_t = f.d_pose_t; a.n_poses = (int)f.n_poses; a.out = f.bm;
  a.counters = (unsigned long long*)f.d_counters;
  // TMA-staged strips (faster than per-lane loads, identical results); the per-lane LDG kernel serves step > 1, the up-down
  // rig, very wide searches and a failed tensor-map encode
  const int strip = c->dc.wx + c->dc.dmax - c->dc.dmin + 15;     // + alignment slack of the box origin
  if (c->dc.step == 1 && !c->dc.updown && c->dc.wy <= 8 && strip <= 112 && c->dc.dmax >= c->dc.dmin) {
    CUtensorMap tm;
    const int bw = strip <= 64 ? 64 : 112;
    if (make_u8_tensor_map(&tm, f.obs_rs, c->dc.W, c->dc.H, c->dc.pitch, bw, c->dc.wy)) {
      if (bw == 64) bm_tma_kernel<64><<<(int)f.n_ev, 32, 0, c->stream>>>(c->dc, a, tm);
      else bm_tma_kernel<112><<<(int)f.n_ev, 32, 0, c->stream>>>(c->dc, a, tm);
      c->launches += 1;
      ESVO_CUDA_TRY(c, cudaGetLastError());
      return ESVO_OK;
    }
  }
  bm_kernel<<<div_up((int)f.n_ev, BM_WARPS), BM_WARPS * 32, 0, c->stream>>>(c->dc, a);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

int seeds_order(Ctx* c) {
  const SlotBufs& f = c->slot();
  if (f.n_ev == 0) return ESVO_OK;          // counters[1] stays 0 from the frame's memset
  seeds_order_kernel<<<div_up((int)f.n_ev, kOrdBlock), kOrdBlock, 0, c->stream>>>(c->dc, f.bm, f.d_ex, f.d_ey, f.d_et, f.d_poses, (int)f.n_ev,
                                                                                f.d_seeds, (unsigned long long*)f.d_counters);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

}  // namespace esvo
