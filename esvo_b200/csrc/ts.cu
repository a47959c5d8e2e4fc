// esvo_b200 product code -- time-surface raster (sm_90a).
//
// Replaces esvo_time_surface::TimeSurface::{eventsCallback, createTimeSurfaceAtTime} and
// EventQueueMat (esvo_time_surface/src/TimeSurface.cpp:52-152,403-425, TimeSurface.h:28-96).
//
// Data layout (HBM, per camera): the event log is SoA (x u16 | y u16 | t i64 | pol u8) in push
// order; the per-pixel deques of the reference are replaced by a "most recent event" index grid:
//   cur_idx[y][x] = max{ i : event i landed on (x,y) }   (atomicMax over 64-bit global indices)
// with its stamp/polarity cached beside it.  For a sync time T newer than every pushed stamp (the
// normal case) this grid IS getMostRecentEventBeforeT.  For an older T the reference semantics are
//   idx = max{ i : pix_i = pix, t_i < T }   valid iff  #{ j : pix_j = pix, t_j >= T } < queue_len
// (events arrive time-ordered, so "t_i < T" is a prefix [0,k) of the log and the deque holds the
// last queue_len arrivals); it is evaluated from the log on the general path below.
// HBM-bound byte work: coalesced SoA reads, one scatter atomic per event, one fused
// decay+convert+median pass over a shared-memory tile, one gather pass for the rectifying remap.
#include "common.cuh"

namespace esvo {

// ---- push: scatter the new events into the incremental grids ----
__global__ void ts_scatter_kernel(const uint16_t* __restrict__ ex, const uint16_t* __restrict__ ey,
                                  const int64_t* __restrict__ et, size_t n, long long gbase, int W, int H,
                                  long long* __restrict__ idx_grid, int32_t* __restrict__ scalars,
                                  long long* __restrict__ max_t) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x = ex[i], y = ey[i];
  long long t = et[i];
  // time-ordered input is required (the reference's insertion sort makes out-of-order input
  // re-insert the globally latest event instead, TimeSurface.cpp:421-422); flag violations.
  if (i > 0 && et[i - 1] > t) scalars[1] = 1;
  if (i == 0 && *max_t > t) scalars[1] = 1;   // max_t is advanced by the second pass, after this kernel
  if (x >= W || y >= H) return;  // EventQueueMat::insideImage
  atomicMax(&idx_grid[(size_t)y * W + x], gbase + (long long)i);
}
// device-resident source: append to the log and scatter in one pass (replaces 4 D2D copies + the scatter kernel)
__global__ void ts_ingest_kernel(const uint16_t* __restrict__ sx, const uint16_t* __restrict__ sy,
                                 const int64_t* __restrict__ st, const uint8_t* __restrict__ sp, size_t n,
                                 uint16_t* __restrict__ ex, uint16_t* __restrict__ ey, int64_t* __restrict__ et,
                                 uint8_t* __restrict__ ep, long long gbase, int W, int H, long long* __restrict__ idx_grid,
                                 int32_t* __restrict__ scalars, const long long* __restrict__ max_t) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = sx[i], y = sy[i];
  const long long t = st[i];
  ex[i] = (uint16_t)x; ey[i] = (uint16_t)y; et[i] = t; ep[i] = sp ? sp[i] : (uint8_t)1;
  if (i > 0 && st[i - 1] > t) scalars[1] = 1;
  if (i == 0 && *max_t > t) scalars[1] = 1;
  if (x >= W || y >= H) return;
  atomicMax(&idx_grid[(size_t)y * W + x], gbase + (long long)i);
}
// ---- packed source: dvs_msgs/Event wire records (common.cuh).  Each warp stages its records through shared memory
// (packed_stage_warp), then each lane decodes its record from there.
// RAW = false: same writes, order flag and scatter as ts_ingest_kernel.  RAW = true: decode into the unordered path's
// raw_* staging only (its run-max kernels do the rest).
template <bool RAW>
__global__ void __launch_bounds__(256) ts_ingest_packed_kernel(const uint8_t* __restrict__ src, size_t n,
                                                               uint16_t* __restrict__ ex, uint16_t* __restrict__ ey,
                                                               int64_t* __restrict__ et, uint8_t* __restrict__ ep, long long gbase,
                                                               int W, int H, long long* __restrict__ idx_grid,
                                                               int32_t* __restrict__ scalars, const long long* __restrict__ max_t) {
  __shared__ uint32_t stage[8][kPackWords];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t i0 = (blockIdx.x * (size_t)blockDim.x) + (size_t)w * 32;   // first record of this warp
  if (i0 >= n) return;
  const size_t i = i0 + lane;
  const uint8_t* r = packed_stage_warp(src, n, i0, lane, stage[w]);
  if (i >= n) return;
  const int x = packed_x(r), y = packed_y(r);
  const long long t = packed_stamp(r);
  const uint8_t pol = r[12] != 0;   // the ROS bool
  ex[i] = (uint16_t)x; ey[i] = (uint16_t)y; et[i] = t; ep[i] = pol;
  if (RAW) return;
  if (i > 0 && packed_stamp(r - kPackRec) > t) scalars[1] = 1;
  if (i == 0 && *max_t > t) scalars[1] = 1;
  if (x >= W || y >= H) return;
  atomicMax(&idx_grid[(size_t)y * W + x], gbase + (long long)i);
}
// second pass: the winner of each pixel caches its stamp and polarity
__global__ void ts_scatter_fix_kernel(const uint16_t* __restrict__ ex, const uint16_t* __restrict__ ey,
                                      const int64_t* __restrict__ et, const uint8_t* __restrict__ ep, size_t n,
                                      long long gbase, int W, int H, const long long* __restrict__ idx_grid,
                                      long long* __restrict__ t_grid, uint8_t* __restrict__ pol_grid,
                                      long long* __restrict__ max_t) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == n - 1 && max_t) atomicMax(max_t, (long long)et[i]);
  int x = ex[i], y = ey[i];
  if (x >= W || y >= H) return;
  size_t p = (size_t)y * W + x;
  if (idx_grid[p] == gbase + (long long)i) { t_grid[p] = et[i]; pol_grid[p] = ep[i]; }
}

// ---- opt-in: stamps out of order.  The reference's eventsCallback (TimeSurface.cpp:403-425) insertion-sorts the new
// event into its global deque and then queues events_.back(), i.e. the event with the LARGEST stamp seen so far (the
// most recent arrival among equal stamps) -- for ordered input that is the new event itself.  So arrival i queues the
// running arg-max of (stamp, arrival) over everything pushed so far: a prefix scan with the associative, non-commutative
// operator  a (+) b = (b.t >= a.t ? b : a).  The effective events are written to the log in arrival order; their stamps
// are non-decreasing, so everything downstream (split by T, queue-length rule, eviction) is unchanged.
struct RunMax { long long t; int i; };
__device__ __forceinline__ RunMax runmax_op(const RunMax& a, const RunMax& b) { return b.t >= a.t ? b : a; }
// (1) per block of 1024 arrivals: inclusive scan -> raw_eff[i] = batch index of the running maximum inside the block;
//     block aggregate -> agg[b] (stamp), agg[nb + b] (batch index)
__global__ void __launch_bounds__(1024) ts_runmax_block_kernel(const int64_t* __restrict__ t, int n, int32_t* __restrict__ eff,
                                                               long long* __restrict__ agg, int nb) {
  __shared__ long long s_t[32];
  __shared__ int s_i[32];
  const int i = blockIdx.x * 1024 + threadIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  RunMax v{i < n ? (long long)t[i] : (long long)0x8000000000000000LL, i < n ? i : -1};
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    RunMax u{__shfl_up_sync(0xffffffffu, v.t, o), __shfl_up_sync(0xffffffffu, v.i, o)};
    if (lane >= o) v = runmax_op(u, v);
  }
  if (lane == 31) { s_t[w] = v.t; s_i[w] = v.i; }
  __syncthreads();
  if (w == 0) {
    RunMax a{s_t[lane], s_i[lane]};
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      RunMax u{__shfl_up_sync(0xffffffffu, a.t, o), __shfl_up_sync(0xffffffffu, a.i, o)};
      if (lane >= o) a = runmax_op(u, a);
    }
    s_t[lane] = a.t; s_i[lane] = a.i;
  }
  __syncthreads();
  if (w > 0) { RunMax pre{s_t[w - 1], s_i[w - 1]}; v = runmax_op(pre, v); }
  if (i < n) eff[i] = v.i;
  if (threadIdx.x == 1023) { agg[blockIdx.x] = v.t; agg[nb + blockIdx.x] = v.i; }
}
// (2) one thread: exclusive scan of the block aggregates seeded with the carried back() event; agg[2nb + b] = stamp and
//     agg[3nb + b] = batch index (-1 = the carried event) of the prefix of block b; back <- new maximum (old one kept)
__global__ void ts_runmax_carry_kernel(long long* agg, int nb, const uint16_t* __restrict__ x, const uint16_t* __restrict__ y,
                                       const int64_t* __restrict__ t, const uint8_t* __restrict__ p, long long* back) {
  if (threadIdx.x || blockIdx.x) return;
  for (int q = 0; q < 5; ++q) back[5 + q] = back[q];
  RunMax run{back[4] ? back[0] : (long long)0x8000000000000000LL, -1};
  for (int b = 0; b < nb; ++b) {
    agg[2 * nb + b] = run.t; agg[3 * nb + b] = run.i;
    run = runmax_op(run, RunMax{agg[b], (int)agg[nb + b]});
  }
  if (run.i >= 0) { back[0] = t[run.i]; back[1] = x[run.i]; back[2] = y[run.i]; back[3] = p ? p[run.i] : 1; back[4] = 1; }
}
// (3) write the effective events to the log and scatter them (same as ts_ingest_kernel on ordered input)
__global__ void ts_effective_kernel(const uint16_t* __restrict__ sx, const uint16_t* __restrict__ sy, const int64_t* __restrict__ st,
                                    const uint8_t* __restrict__ sp, int n, const int32_t* __restrict__ eff,
                                    const long long* __restrict__ agg, int nb, const long long* __restrict__ back,
                                    uint16_t* __restrict__ ex, uint16_t* __restrict__ ey, int64_t* __restrict__ et, uint8_t* __restrict__ ep,
                                    long long gbase, int W, int H, long long* __restrict__ idx_grid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = i >> 10;
  int j = eff[i];
  const long long pre_t = agg[2 * nb + b];
  const int pre_i = (int)agg[3 * nb + b];
  const bool have_pre = pre_i >= 0 || back[5 + 4] != 0;
  if (have_pre && !((long long)st[j] >= pre_t)) j = pre_i;    // the prefix (earlier arrivals) holds a strictly later stamp
  int x, y; long long t; int pol;
  if (j >= 0) { x = sx[j]; y = sy[j]; t = st[j]; pol = sp ? sp[j] : 1; }
  else { t = back[5]; x = (int)back[6]; y = (int)back[7]; pol = (int)back[8]; }   // the event carried over from earlier pushes
  ex[i] = (uint16_t)x; ey[i] = (uint16_t)y; et[i] = t; ep[i] = (uint8_t)pol;
  if (x >= W || y >= H) return;
  atomicMax(&idx_grid[(size_t)y * W + x], gbase + (long long)i);
}

// ---- build, step 0: split position k = first log entry with t >= T; flag the general path ----
// Folded into the first general-path kernel: thread 0 of every block runs the (L2-resident, ~22-step) binary search
// itself, block 0 publishes the result for the kernels that follow.  One launch less on the serial TS chain.
__device__ __forceinline__ void ts_split_block(const int64_t* __restrict__ et, size_t n, long long T, int32_t* scalars,
                                               int& k_out, int& general_out) {
  __shared__ int s_k, s_general;
  if (threadIdx.x == 0) {
    size_t lo = 0, hi = n;
    while (lo < hi) { size_t mid = (lo + hi) >> 1; if (et[mid] < T) lo = mid + 1; else hi = mid; }
    s_k = (int)lo; s_general = (lo != n) ? 1 : 0;
    if (blockIdx.x == 0) { scalars[0] = s_k; scalars[2] = s_general; }
  }
  __syncthreads();
  k_out = s_k; general_out = s_general;
}
// general path (no-ops when scalars[2]==0)
__global__ void ts_general_init_kernel(int32_t* scalars, const int64_t* __restrict__ et, size_t log_n, long long T, size_t npix,
                                       const long long* __restrict__ bidx, const long long* __restrict__ bt,
                                       const uint8_t* __restrict__ bpol, long long* tidx, long long* tt, uint8_t* tpol, int32_t* cnt) {
  int k, general;
  ts_split_block(et, log_n, T, scalars, k, general);
  if (!general) return;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
    tidx[i] = bidx[i]; tt[i] = bt[i]; tpol[i] = bpol[i]; cnt[i] = 0;
  }
}
__global__ void ts_general_scatter_kernel(const int32_t* __restrict__ scalars, const uint16_t* __restrict__ ex,
                                          const uint16_t* __restrict__ ey, size_t n, long long gbase, int W, int H,
                                          long long* tidx, int32_t* cnt) {
  if (!scalars[2]) return;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    int x = ex[i], y = ey[i];
    if (x >= W || y >= H) continue;
    size_t p = (size_t)y * W + x;
    if (i < (size_t)scalars[0]) atomicMax(&tidx[p], gbase + (long long)i);
    else atomicAdd(&cnt[p], 1);
  }
}
__global__ void ts_general_fix_kernel(const int32_t* __restrict__ scalars, const uint16_t* __restrict__ ex,
                                      const uint16_t* __restrict__ ey, const int64_t* __restrict__ et,
                                      const uint8_t* __restrict__ ep, size_t n, long long gbase, int W, int H,
                                      const long long* tidx, long long* tt, uint8_t* tpol) {
  if (!scalars[2]) return;
  const size_t k = (size_t)scalars[0];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < k; i += (size_t)gridDim.x * blockDim.x) {
    int x = ex[i], y = ey[i];
    if (x >= W || y >= H) continue;
    size_t p = (size_t)y * W + x;
    if (tidx[p] == gbase + (long long)i) { tt[p] = et[i]; tpol[p] = ep[i]; }
  }
}

// ---- build, step 1: decay + u8 convert + 3x3 median, fused over a shared-memory tile ----
constexpr int TSX = 32, TSY = 8;
__device__ __forceinline__ void sort2(int& a, int& b) { int lo = min(a, b), hi = max(a, b); a = lo; b = hi; }

template <int KS>
__global__ void ts_decay_median_kernel(const int32_t* __restrict__ scalars, const long long* __restrict__ cur_idx,
                                       const long long* __restrict__ cur_t, const uint8_t* __restrict__ cur_pol,
                                       const long long* __restrict__ tmp_idx, const long long* __restrict__ tmp_t,
                                       const uint8_t* __restrict__ tmp_pol, const int32_t* __restrict__ cnt,
                                       int queue_len, long long T, double decay_sec, int ignore_polarity, int W, int H,
                                       int pitch, long long* __restrict__ out_idx, uint8_t* __restrict__ img, int maybe_general) {
  constexpr int R = KS / 2;
  __shared__ uint8_t tile[TSY + 2 * R][TSX + 2 * R + 2];
  const bool general = maybe_general && scalars[2] != 0;   // maybe_general == 0: the host knows T is newer than every stamp
  const long long* gi = general ? tmp_idx : cur_idx;
  const long long* gt = general ? tmp_t : cur_t;
  const uint8_t* gp = general ? tmp_pol : cur_pol;
  const int x0 = blockIdx.x * TSX, y0 = blockIdx.y * TSY;
  for (int k = threadIdx.y * TSX + threadIdx.x; k < (TSY + 2 * R) * (TSX + 2 * R); k += TSX * TSY) {
    int ty = k / (TSX + 2 * R), tx = k % (TSX + 2 * R);
    int gx = min(max(x0 + tx - R, 0), W - 1), gy = min(max(y0 + ty - R, 0), H - 1);  // BORDER_REPLICATE
    size_t p = (size_t)gy * W + gx;
    long long idx = gi[p];
    if (general && idx >= 0 && cnt[p] >= queue_len) idx = -1;   // fell out of the 20-deep queue
    double v = 0.0;
    long long ts = idx >= 0 ? gt[p] : 0;
    if (idx >= 0 && !(ns_to_sec_dev(ts) > 0)) idx = -1;          // TimeSurface.cpp:73
    if (idx >= 0) {
      double dt = ns_to_sec_dev(T - ts);
      v = exp(-dt / decay_sec);                                  // :77
      if (!ignore_polarity) v *= gp[p] ? 1.0 : -1.0;
    }
    if (tx >= R && tx < TSX + R && ty >= R && ty < TSY + R && x0 + tx - R < W && y0 + ty - R < H)
      out_idx[(size_t)(y0 + ty - R) * W + x0 + tx - R] = idx;
    double s = ignore_polarity ? 255.0 * v : 255.0 * (v + 1.0) / 2.0;  // :123-126
    int r = __double2int_rn(s);                                        // cvRound, half-to-even
    tile[ty][tx] = (uint8_t)min(max(r, 0), 255);
  }
  __syncthreads();
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= W || y >= H) return;
  int out;
  if (KS == 1) out = tile[threadIdx.y][threadIdx.x];
  else {
    // 3x3 median by the classic 19-exchange network
    int p0 = tile[threadIdx.y][threadIdx.x], p1 = tile[threadIdx.y][threadIdx.x + 1], p2 = tile[threadIdx.y][threadIdx.x + 2];
    int p3 = tile[threadIdx.y + 1][threadIdx.x], p4 = tile[threadIdx.y + 1][threadIdx.x + 1], p5 = tile[threadIdx.y + 1][threadIdx.x + 2];
    int p6 = tile[threadIdx.y + 2][threadIdx.x], p7 = tile[threadIdx.y + 2][threadIdx.x + 1], p8 = tile[threadIdx.y + 2][threadIdx.x + 2];
    sort2(p1, p2); sort2(p4, p5); sort2(p7, p8); sort2(p0, p1); sort2(p3, p4); sort2(p6, p7);
    sort2(p1, p2); sort2(p4, p5); sort2(p7, p8); sort2(p0, p3); sort2(p5, p8); sort2(p4, p7);
    sort2(p3, p6); sort2(p1, p4); sort2(p2, p5); sort2(p4, p7); sort2(p4, p2); sort2(p6, p4);
    sort2(p4, p2);
    out = p4;
  }
  img[(size_t)y * pitch + x] = (uint8_t)out;
}

// ---- build, step 2: rectifying remap (cv::remap INTER_LINEAR, 1/32-px fixed point, border 0) ----
__global__ void ts_remap_kernel(const uint8_t* __restrict__ src, const float* __restrict__ map1,
                                const float* __restrict__ map2, int W, int H, int pitch, uint8_t* __restrict__ dst) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  size_t i = (size_t)y * W + x;
  int sx = __float2int_rn(__fmul_rn(map1[i], 32.0f)), sy = __float2int_rn(__fmul_rn(map2[i], 32.0f));
  int fx = sx & 31, fy = sy & 31;
  int ix = min(max(sx >> 5, -32768), 32767), iy = min(max(sy >> 5, -32768), 32767);
  auto px = [&](int xx, int yy) -> int {
    return (xx >= 0 && xx < W && yy >= 0 && yy < H) ? (int)src[(size_t)yy * pitch + xx] : 0;
  };
  int v = 32 * (32 - fx) * (32 - fy) * px(ix, iy) + 32 * fx * (32 - fy) * px(ix + 1, iy) +
          32 * (32 - fx) * fy * px(ix, iy + 1) + 32 * fx * fy * px(ix + 1, iy + 1);
  dst[(size_t)y * pitch + x] = (uint8_t)((v + (1 << 14)) >> 15);
}
// ---- FORWARD mode (TimeSurface.cpp:86-116): every raw pixel splats its decayed value bilinearly onto the four
// rectified neighbours, each accumulation followed by a clamp at 1.  The reference walks the raw image in raster
// order, and v <- min(v + w, 1) does not commute, so the result at a destination depends on the ORDER of the
// sources that reach it (not on anything else).  Same scheme as the depth fusion: (1) one thread per source appends
// its four contributions to per-destination linked lists (one atomicExch each), node id = 4*source + corner;
// (2) one thread per destination replays its list in ascending node id = raster order of the sources.
__global__ void ts_forward_scatter_kernel(const int32_t* __restrict__ scalars, const long long* __restrict__ cur_idx,
                                          const long long* __restrict__ cur_t, const uint8_t* __restrict__ cur_pol,
                                          const long long* __restrict__ tmp_idx, const long long* __restrict__ tmp_t,
                                          const uint8_t* __restrict__ tmp_pol, const int32_t* __restrict__ cnt, int queue_len,
                                          long long T, double decay_sec, int ignore_polarity, int W, int H,
                                          const double* __restrict__ lut, long long* __restrict__ out_idx,
                                          int32_t* head, int32_t* __restrict__ next, double* __restrict__ val, int maybe_general) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= W * H) return;
  const bool general = maybe_general && scalars[2] != 0;
  long long idx = general ? tmp_idx[p] : cur_idx[p];
  if (general && idx >= 0 && cnt[p] >= queue_len) idx = -1;   // fell out of the 20-deep queue
  const long long ts = idx >= 0 ? (general ? tmp_t[p] : cur_t[p]) : 0;
  if (idx >= 0 && !(ns_to_sec_dev(ts) > 0)) idx = -1;          // :73
  out_idx[p] = idx;
  if (idx < 0) return;
  const double dt = ns_to_sec_dev(T - ts);
  double e = exp(-dt / decay_sec);                             // :77
  if (!ignore_polarity) e *= (general ? tmp_pol[p] : cur_pol[p]) ? 1.0 : -1.0;
  const double u = lut[2 * (size_t)p], v = lut[2 * (size_t)p + 1];
  if (!(u >= 0 && v >= 0)) return;                             // :89 (NaN fails the test like in the reference)
  if (u >= (double)W || v >= (double)H) return;                // u_i + 1 < W cannot hold; also keeps floor() in int range
  const int ui = (int)floor(u), vi = (int)floor(v);
  if (!(ui + 1 < W && vi + 1 < H)) return;                     // :94
  const double fu = u - ui, fv = v - vi, fu1 = 1.0 - fu, fv1 = 1.0 - fv;
  const double w[4] = {fu1 * fv1 * e, fu * fv1 * e, fu1 * fv * e, fu * fv * e};
  const int dst[4] = {vi * W + ui, vi * W + ui + 1, (vi + 1) * W + ui, (vi + 1) * W + ui + 1};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int node = 4 * p + k;
    val[node] = w[k];
    next[node] = atomicExch(&head[dst[k]], node);
  }
}
__global__ void ts_forward_fold_kernel(int W, int H, int pitch, int32_t* head, const int32_t* __restrict__ next,
                                       const double* __restrict__ val, int ignore_polarity, uint8_t* __restrict__ img) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= W * H) return;
  const int h = head[p];
  head[p] = -1;
  constexpr int CAP = 32;
  int ids[CAP];
  int n = 0, total = 0;
  for (int q = h; q >= 0; q = next[q]) { if (n < CAP) ids[n++] = q; ++total; }
  double m = 0.0;
  if (total <= CAP) {
    for (int a = 1; a < n; ++a) { int v = ids[a], b = a - 1; while (b >= 0 && ids[b] > v) { ids[b + 1] = ids[b]; --b; } ids[b + 1] = v; }
    for (int a = 0; a < n; ++a) { m += val[ids[a]]; if (m > 1) m = 1; }        // :101-113
  } else {   // very long list: repeated minimum selection, no storage
    int last = -1;
    for (int a = 0; a < total; ++a) {
      int best = 0x7fffffff;
      for (int q = h; q >= 0; q = next[q]) if (q > last && q < best) best = q;
      m += val[best]; if (m > 1) m = 1;
      last = best;
    }
  }
  const double s = ignore_polarity ? 255.0 * m : 255.0 * (m + 1.0) / 2.0;   // :123-126
  const int r = __double2int_rn(s);                                         // cvRound, half-to-even
  const int y = p / W, x = p - y * W;
  img[(size_t)y * pitch + x] = (uint8_t)min(max(r, 0), 255);
}
// cv::medianBlur 3x3 on u8, BORDER_REPLICATE
__global__ void ts_median3_kernel(const uint8_t* __restrict__ src, int W, int H, int pitch, uint8_t* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  int v[9];
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx)
      v[(dy + 1) * 3 + dx + 1] = src[(size_t)min(max(y + dy, 0), H - 1) * pitch + min(max(x + dx, 0), W - 1)];
  sort2(v[1], v[2]); sort2(v[4], v[5]); sort2(v[7], v[8]); sort2(v[0], v[1]); sort2(v[3], v[4]); sort2(v[6], v[7]);
  sort2(v[1], v[2]); sort2(v[4], v[5]); sort2(v[7], v[8]); sort2(v[0], v[3]); sort2(v[5], v[8]); sort2(v[4], v[7]);
  sort2(v[3], v[6]); sort2(v[1], v[4]); sort2(v[2], v[5]); sort2(v[4], v[7]); sort2(v[4], v[2]); sort2(v[6], v[4]);
  sort2(v[4], v[2]);
  dst[(size_t)y * pitch + x] = (uint8_t)v[4];
}
__global__ void fill_i32_ts_kernel(int32_t* p, size_t n, int32_t v) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void ts_copy_img_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}
__global__ void fill_i64_kernel(long long* p, size_t n, long long v) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// --------------------------------------------------------------------------------------------

int ts_reset_state(Ctx* c, int cam) {
  TsState& s = c->ts[cam];
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  const int B = 256;
  fill_i64_kernel<<<(unsigned)((npix + B - 1) / B), B, 0, c->stream>>>((long long*)s.cur_idx, npix, -1);
  fill_i64_kernel<<<(unsigned)((npix + B - 1) / B), B, 0, c->stream>>>((long long*)s.base_idx, npix, -1);
  c->launches += 2;
  ESVO_CUDA_TRY(c, cudaMemsetAsync(s.cur_t, 0, npix * 8, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(s.base_t, 0, npix * 8, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(s.cur_pol, 0, npix, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(s.base_pol, 0, npix, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(s.scalars, 0, 16 * sizeof(int32_t), c->stream));
  long long mn = INT64_MIN;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.max_t, &mn, 8, cudaMemcpyHostToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(s.img_out, 0, (size_t)c->dc.pitch * c->dc.H, c->stream));
  if (s.back) ESVO_CUDA_TRY(c, cudaMemsetAsync(s.back, 0, 80, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  s.log_n = 0; s.log_base = 0; s.built = false; s.last_img = s.img_out;
  s.host_knows = true; s.host_max_t = INT64_MIN;
  return ESVO_OK;
}

int ts_alloc(Ctx* c, int cam) {
  TsState& s = c->ts[cam];
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  s.log_cap = (size_t)1 << 22;  // 4 Mi events resident per camera (2 x 52 MiB, ping-pong); older ones fold into base grids
  ESVO_CUDA_TRY(c, dmalloc(&s.ex, s.log_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.ey, s.log_cap));
  ESVO_CUDA_TRY(c, dmalloc(&s.et, s.log_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.ep, s.log_cap));
  ESVO_CUDA_TRY(c, dmalloc(&s.ex2, s.log_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.ey2, s.log_cap));
  ESVO_CUDA_TRY(c, dmalloc(&s.et2, s.log_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.ep2, s.log_cap));
  ESVO_CUDA_TRY(c, dmalloc(&s.cur_idx, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.cur_t, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.cur_pol, npix));
  ESVO_CUDA_TRY(c, dmalloc(&s.base_idx, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.base_t, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.base_pol, npix));
  ESVO_CUDA_TRY(c, dmalloc(&s.tmp_idx, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.tmp_t, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.tmp_pol, npix));
  ESVO_CUDA_TRY(c, dmalloc(&s.cnt, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.out_idx, npix));
  ESVO_CUDA_TRY(c, dmalloc(&s.img_med, (size_t)c->dc.pitch * c->dc.H));
  ESVO_CUDA_TRY(c, dmalloc(&s.img_out, (size_t)c->dc.pitch * c->dc.H));
  ESVO_CUDA_TRY(c, dmalloc(&s.map1, npix)); ESVO_CUDA_TRY(c, dmalloc(&s.map2, npix));
  ESVO_CUDA_TRY(c, dmalloc(&s.scalars, 16)); ESVO_CUDA_TRY(c, dmalloc(&s.max_t, 1));
  ESVO_CUDA_TRY(c, cudaMemcpy(s.map1, c->cam[cam].map1.data(), npix * 4, cudaMemcpyHostToDevice));
  ESVO_CUDA_TRY(c, cudaMemcpy(s.map2, c->cam[cam].map2.data(), npix * 4, cudaMemcpyHostToDevice));
  ESVO_CUDA_TRY(c, cudaMemset(s.img_med, 0, (size_t)c->dc.pitch * c->dc.H));
  return ts_reset_state(c, cam);
}
void ts_free(Ctx* c, int cam) {
  TsState& s = c->ts[cam];
  void* ps[] = {s.ex2, s.ey2, s.et2, s.ep2, s.ex, s.ey, s.et, s.ep, s.cur_idx, s.cur_t, s.cur_pol, s.base_idx, s.base_t, s.base_pol, s.tmp_idx,
                s.tmp_t, s.tmp_pol, s.cnt, s.out_idx, s.img_med, s.img_out, s.map1, s.map2, s.scalars, s.max_t,
                s.fwd_lut, s.fwd_head, s.fwd_next, s.fwd_val, s.raw_x, s.raw_y, s.raw_t, s.raw_p, s.raw_eff, s.agg, s.back, s.pack_dev};
  for (void* p : ps) if (p) cudaFree(p);
  if (s.h_pack) cudaFreeHost(s.h_pack);
  if (s.ev_pack) cudaEventDestroy(s.ev_pack);
  hp_free(s);
  s = TsState();
}

// When the next push would overflow the resident log, fold the oldest events into the base grids and
// move the most recent ones to the alternate buffer set (ping-pong).  Everything is enqueued on the
// ctx stream: no allocation, no host synchronisation.
static int ts_make_room(Ctx* c, int cam, size_t n_new) {
  TsState& s = c->ts[cam];
  if (n_new > s.log_cap / 2) { c->set_error("event batch larger than half the resident log"); return ESVO_ERR_CAPACITY; }
  if (s.log_n + n_new <= s.log_cap) return ESVO_OK;
  const size_t keep = std::min(s.log_n, s.log_cap / 4);
  const size_t drop = s.log_n - keep;
  const int B = 256;
  unsigned g = (unsigned)((drop + B - 1) / B);
  // scalars[12..13] (one int64): stamp of the first event ever pushed, which the first fold is about to drop.  With the newest
  // folded stamp it bounds every folded stamp (events.cu answers some lower bounds into the folded part from the two).
  if (s.log_base == 0) ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.scalars + 12, s.et, 8, cudaMemcpyDeviceToDevice, c->stream));
  ts_scatter_kernel<<<g, B, 0, c->stream>>>(s.ex, s.ey, s.et, drop, s.log_base, c->dc.W, c->dc.H, (long long*)s.base_idx,
                                            s.scalars + 8, (long long*)(s.max_t));
  // scalars[10..11] (one int64): stamp of the newest folded event.  A build at T <= that stamp cannot be answered any more
  // (folded events with t >= T are neither counted against the queue length nor skipped); esvo_ts_build refuses it.
  ts_scatter_fix_kernel<<<g, B, 0, c->stream>>>(s.ex, s.ey, s.et, s.ep, drop, s.log_base, c->dc.W, c->dc.H,
                                                (const long long*)s.base_idx, (long long*)s.base_t, s.base_pol,
                                                (long long*)(s.scalars + 10));
  c->launches += 2;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.ex2, s.ex + drop, keep * 2, cudaMemcpyDeviceToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.ey2, s.ey + drop, keep * 2, cudaMemcpyDeviceToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.et2, s.et + drop, keep * 8, cudaMemcpyDeviceToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.ep2, s.ep + drop, keep, cudaMemcpyDeviceToDevice, c->stream));
  std::swap(s.ex, s.ex2); std::swap(s.ey, s.ey2); std::swap(s.et, s.et2); std::swap(s.ep, s.ep2);
  s.log_base += (int64_t)drop; s.log_n = keep;
  return ESVO_OK;
}

// x/y/t/p are HOST pointers; the copies are enqueued on the ctx stream (pageable memory is staged
// by the driver; callers that want true async overlap pass pinned buffers).
// Host event packet whose four arrays are adjacent (at most 64 bytes of padding in total): start of the span, else null.
static const uint8_t* packet_span(const uint16_t* x, const uint16_t* y, const int64_t* t, const uint8_t* p, size_t n, size_t& span) {
  if (!p || n < 4096) return nullptr;                    // small pushes: the copies are not what costs
  const uint8_t* b[4] = {(const uint8_t*)x, (const uint8_t*)y, (const uint8_t*)t, p};
  const size_t len[4] = {n * 2, n * 2, n * 8, n};
  const uint8_t *lo = b[0], *hi = b[0] + len[0];
  for (int i = 1; i < 4; ++i) { if (b[i] < lo) lo = b[i]; if (b[i] + len[i] > hi) hi = b[i] + len[i]; }
  span = (size_t)(hi - lo);
  return span <= n * 13 + 64 ? lo : nullptr;
}

// Unordered input (esvo_ts_set_unordered_input): the raw batch staging, block aggregates and carried event, grown to n.
static int ts_raw_reserve(Ctx* c, TsState& s, size_t n) {
  const int nb = (int)((n + 1023) / 1024);
  if (!s.back) { ESVO_CUDA_TRY(c, dmalloc(&s.back, 10)); ESVO_CUDA_TRY(c, cudaMemsetAsync(s.back, 0, 80, c->stream)); }
  if (n > s.raw_cap) {
    ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    void* olds[] = {s.raw_x, s.raw_y, s.raw_t, s.raw_p, s.raw_eff};
    for (void* q : olds) if (q) cudaFree(q);
    s.raw_cap = std::max<size_t>(n, 1 << 16);
    ESVO_CUDA_TRY(c, dmalloc(&s.raw_x, s.raw_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.raw_y, s.raw_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.raw_t, s.raw_cap));
    ESVO_CUDA_TRY(c, dmalloc(&s.raw_p, s.raw_cap)); ESVO_CUDA_TRY(c, dmalloc(&s.raw_eff, s.raw_cap));
  }
  if ((size_t)nb * 4 > s.agg_cap) {
    ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (s.agg) cudaFree(s.agg);
    s.agg_cap = std::max<size_t>((size_t)nb * 4, 1024);
    ESVO_CUDA_TRY(c, dmalloc(&s.agg, s.agg_cap));
  }
  return ESVO_OK;
}
// Unordered input: the running arg-max of the stamps picks each arrival's effective event, which goes to the log at off.
static void ts_runmax_push(Ctx* c, TsState& s, const uint16_t* sx, const uint16_t* sy, const int64_t* st, const uint8_t* sp, size_t n,
                           size_t off, long long gbase) {
  const int nb = (int)((n + 1023) / 1024), B = 256;
  const unsigned g = (unsigned)((n + B - 1) / B);
  ts_runmax_block_kernel<<<nb, 1024, 0, c->stream>>>(st, (int)n, s.raw_eff, (long long*)s.agg, nb);
  ts_runmax_carry_kernel<<<1, 32, 0, c->stream>>>((long long*)s.agg, nb, sx, sy, st, sp, (long long*)s.back);
  ts_effective_kernel<<<g, B, 0, c->stream>>>(sx, sy, st, sp, (int)n, s.raw_eff, (const long long*)s.agg, nb, (const long long*)s.back,
                                              s.ex + off, s.ey + off, s.et + off, s.ep + off, gbase, c->dc.W, c->dc.H, (long long*)s.cur_idx);
  c->launches += 3;
}

int ts_push(Ctx* c, int cam, const uint16_t* x, const uint16_t* y, const int64_t* t, const uint8_t* p, size_t n, bool dev_src) {
  if (n == 0) return ESVO_OK;
  size_t span = 0;
  TsState& s = c->ts[cam];
  int rc = ts_make_room(c, cam, n);
  if (rc) return rc;
  size_t off = s.log_n;
  cudaEvent_t pe = c->prof_begin(0);
  const int B = 256;
  unsigned g = (unsigned)((n + B - 1) / B);
  long long gbase = s.log_base + (long long)off;
  if (dev_src || s.unordered) s.host_knows = false;
  else if (s.host_knows) { if (t[n - 1] >= s.host_max_t) s.host_max_t = t[n - 1]; else s.host_knows = false; }
  if (s.unordered) {
    if ((rc = ts_raw_reserve(c, s, n))) return rc;
    const uint16_t *sx = x, *sy = y; const int64_t* st = t; const uint8_t* sp = p;
    if (!dev_src) {
      ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.raw_x, x, n * 2, cudaMemcpyHostToDevice, c->stream));
      ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.raw_y, y, n * 2, cudaMemcpyHostToDevice, c->stream));
      ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.raw_t, t, n * 8, cudaMemcpyHostToDevice, c->stream));
      if (p) ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.raw_p, p, n, cudaMemcpyHostToDevice, c->stream));
      sx = s.raw_x; sy = s.raw_y; st = s.raw_t; sp = p ? s.raw_p : nullptr;
    }
    ts_runmax_push(c, s, sx, sy, st, sp, n, off, gbase);
  } else if (dev_src) {
    ts_ingest_kernel<<<g, B, 0, c->stream>>>(x, y, t, p, n, s.ex + off, s.ey + off, s.et + off, s.ep + off, gbase, c->dc.W, c->dc.H,
                                             (long long*)s.cur_idx, s.scalars, (const long long*)s.max_t);
  } else if (const uint8_t* lo = packet_span(x, y, t, p, n, span)) {
    // The four arrays sit next to each other in host memory (one packet buffer, e.g. t | x | y | p): ONE copy of the whole
    // span into a landing buffer (same address skew mod 16, so every array keeps its alignment), then the device-source
    // ingest kernel.  Three copies fewer per push -- the host-buffer path is host-issue-bound (DESIGN.md 9).
    const size_t skew = (size_t)((uintptr_t)lo & 15);
    if (span + 16 > s.pack_cap) {
      ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
      if (s.pack_dev) cudaFree(s.pack_dev);
      s.pack_cap = std::max<size_t>(2 * (span + 16), (size_t)1 << 20);
      ESVO_CUDA_TRY(c, dmalloc(&s.pack_dev, s.pack_cap));
    }
    uint8_t* d0 = s.pack_dev + skew;
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(d0, lo, span, cudaMemcpyHostToDevice, c->stream));
    ts_ingest_kernel<<<g, B, 0, c->stream>>>((const uint16_t*)(d0 + ((const uint8_t*)x - lo)), (const uint16_t*)(d0 + ((const uint8_t*)y - lo)),
                                             (const int64_t*)(d0 + ((const uint8_t*)t - lo)), d0 + (p - lo), n, s.ex + off, s.ey + off, s.et + off,
                                             s.ep + off, gbase, c->dc.W, c->dc.H, (long long*)s.cur_idx, s.scalars, (const long long*)s.max_t);
  } else {
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.ex + off, x, n * 2, cudaMemcpyHostToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.ey + off, y, n * 2, cudaMemcpyHostToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.et + off, t, n * 8, cudaMemcpyHostToDevice, c->stream));
    if (p) ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.ep + off, p, n, cudaMemcpyHostToDevice, c->stream));
    else ESVO_CUDA_TRY(c, cudaMemsetAsync(s.ep + off, 1, n, c->stream));
    ts_scatter_kernel<<<g, B, 0, c->stream>>>(s.ex + off, s.ey + off, s.et + off, n, gbase, c->dc.W, c->dc.H,
                                              (long long*)s.cur_idx, s.scalars, (long long*)s.max_t);
  }
  ts_scatter_fix_kernel<<<g, B, 0, c->stream>>>(s.ex + off, s.ey + off, s.et + off, s.ep + off, n, gbase, c->dc.W, c->dc.H,
                                                (const long long*)s.cur_idx, (long long*)s.cur_t, s.cur_pol, (long long*)s.max_t);
  c->launches += 2;
  c->prof_end(pe);
  s.log_n += n;
  return ESVO_OK;
}

// n dvs_msgs/Event wire records (13 bytes each, any alignment) in device memory.  Everything after the decode is ts_push's:
// the same log, push indices, order flag, fold and refusals.  host_last_t: the stamp of the last record when the host knows
// it (the host form below), else null -- as for ts_push's host and device sources.
// With a hot-pixel mask installed (esvo_hotpix_select) the records at hot pixels are dropped first (hp_compact_packed, one
// read-back of the number kept and the last kept stamp) and the push continues on the kept records, with that stamp as
// host_last_t.  The half-log refusal applies to the n records handed in, before the filter.
int ts_push_packed(Ctx* c, int cam, const uint8_t* src, size_t n, const int64_t* host_last_t) {
  if (n == 0) return ESVO_OK;
  TsState& s = c->ts[cam];
  int rc;
  int64_t kept_last_t;
  if (s.hp.masked) {
    if (n > s.log_cap / 2) { c->set_error("event batch larger than half the resident log"); return ESVO_ERR_CAPACITY; }
    if ((rc = hp_compact_packed(c, cam, src, n, &src, &n, &kept_last_t))) return rc;
    if (n == 0) return ESVO_OK;
    host_last_t = &kept_last_t;
  }
  rc = ts_make_room(c, cam, n);
  if (rc) return rc;
  const size_t off = s.log_n;
  cudaEvent_t pe = c->prof_begin(0);
  const int B = 256;
  const unsigned g = (unsigned)((n + B - 1) / B);
  const long long gbase = s.log_base + (long long)off;
  if (!host_last_t || s.unordered) s.host_knows = false;
  else if (s.host_knows) { if (*host_last_t >= s.host_max_t) s.host_max_t = *host_last_t; else s.host_knows = false; }
  if (s.unordered) {
    if ((rc = ts_raw_reserve(c, s, n))) return rc;
    ts_ingest_packed_kernel<true><<<g, B, 0, c->stream>>>(src, n, s.raw_x, s.raw_y, s.raw_t, s.raw_p, gbase, c->dc.W, c->dc.H, nullptr,
                                                          nullptr, nullptr);
    c->launches += 1;
    ts_runmax_push(c, s, s.raw_x, s.raw_y, s.raw_t, s.raw_p, n, off, gbase);
  } else {
    ts_ingest_packed_kernel<false><<<g, B, 0, c->stream>>>(src, n, s.ex + off, s.ey + off, s.et + off, s.ep + off, gbase, c->dc.W,
                                                           c->dc.H, (long long*)s.cur_idx, s.scalars, (const long long*)s.max_t);
  }
  ts_scatter_fix_kernel<<<g, B, 0, c->stream>>>(s.ex + off, s.ey + off, s.et + off, s.ep + off, n, gbase, c->dc.W, c->dc.H,
                                                (const long long*)s.cur_idx, (long long*)s.cur_t, s.cur_pol, (long long*)s.max_t);
  c->launches += 2;
  c->prof_end(pe);
  s.log_n += n;
  return ESVO_OK;
}

// The pinned staging block of camera cam and its device landing buffer, both at least `bytes` long, once the previous copy
// out of the staging block has completed.
int ts_pack_staging(Ctx* c, int cam, size_t bytes) {
  TsState& s = c->ts[cam];
  if (s.ev_pack) ESVO_CUDA_TRY(c, cudaEventSynchronize(s.ev_pack));
  else ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&s.ev_pack, cudaEventDisableTiming));
  if (bytes > s.h_pack_cap) {
    if (s.h_pack) cudaFreeHost(s.h_pack);
    s.h_pack = nullptr;
    s.h_pack_cap = std::max<size_t>(2 * bytes, (size_t)1 << 20);
    ESVO_CUDA_TRY(c, cudaMallocHost((void**)&s.h_pack, s.h_pack_cap));
  }
  if (bytes > s.pack_cap) {
    ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (s.pack_dev) cudaFree(s.pack_dev);
    s.pack_dev = nullptr;
    s.pack_cap = std::max<size_t>(2 * bytes, (size_t)1 << 20);
    ESVO_CUDA_TRY(c, dmalloc(&s.pack_dev, s.pack_cap));
  }
  return ESVO_OK;
}

// Host runs of wire records (e.g. the event blocks of several EventArray messages in a memory-mapped bag): gathered with
// memcpy into this camera's pinned staging block, one H2D copy, then ts_push_packed on the copy.  The staging block is
// reused once the previous copy out of it has completed, so the caller's runs are free again on return.
int ts_push_packed_host(Ctx* c, int cam, const uint8_t* const* runs, const size_t* n_events, int n_runs) {
  TsState& s = c->ts[cam];
  size_t n = 0;
  for (int k = 0; k < n_runs; ++k) n += n_events[k];
  if (n == 0) return ESVO_OK;
  if (n > s.log_cap / 2) { c->set_error("event batch larger than half the resident log"); return ESVO_ERR_CAPACITY; }
  const size_t bytes = n * kPackRec;
  int rc = ts_pack_staging(c, cam, bytes);
  if (rc) return rc;
  uint8_t* d = s.h_pack;
  for (int k = 0; k < n_runs; ++k) {
    if (!n_events[k]) continue;
    std::memcpy(d, runs[k], n_events[k] * kPackRec);
    d += n_events[k] * kPackRec;
  }
  const uint8_t* last = d - kPackRec;
  uint32_t sec, nsec;
  std::memcpy(&sec, last + 4, 4); std::memcpy(&nsec, last + 8, 4);
  const int64_t t_last = (int64_t)sec * 1000000000LL + (int64_t)nsec;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.pack_dev, s.h_pack, bytes, cudaMemcpyHostToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaEventRecord(s.ev_pack, c->stream));
  return ts_push_packed(c, cam, s.pack_dev, n, &t_last);
}

int ts_run_build(Ctx* c, int cam, int64_t T) {
  TsState& s = c->ts[cam];
  const DevConsts& d = c->dc;
  const size_t npix = (size_t)d.W * d.H;
  const int B = 256;
  cudaEvent_t pe = c->prof_begin(0);
  const unsigned GG = c->num_sms * 4;   // fixed grid, grid-stride loops: these three kernels are no-ops on the fast path
  // T newer than every pushed stamp (known on the host for host-buffer pushes of ordered input): the most-recent-event grid
  // IS the answer and the general path's three launches (no-ops on the device in that case) are not issued at all
  const int maybe_general = (s.host_knows && (s.log_n == 0 || T > s.host_max_t)) ? 0 : 1;
  if (maybe_general) {
    ts_general_init_kernel<<<GG, B, 0, c->stream>>>(
        s.scalars, s.et, s.log_n, T, npix, (const long long*)s.base_idx, (const long long*)s.base_t, s.base_pol, (long long*)s.tmp_idx,
        (long long*)s.tmp_t, s.tmp_pol, s.cnt);
    c->launches += 1;
  }
  if (maybe_general && s.log_n) {
    ts_general_scatter_kernel<<<GG, B, 0, c->stream>>>(s.scalars, s.ex, s.ey, s.log_n, s.log_base, d.W, d.H,
                                                      (long long*)s.tmp_idx, s.cnt);
    ts_general_fix_kernel<<<GG, B, 0, c->stream>>>(s.scalars, s.ex, s.ey, s.et, s.ep, s.log_n, s.log_base, d.W, d.H,
                                                  (const long long*)s.tmp_idx, (long long*)s.tmp_t, s.tmp_pol);
    c->launches += 2;
  }
  dim3 blk(TSX, TSY), grd(div_up(d.W, TSX), div_up(d.H, TSY));
  const double decay_sec = c->prm.decay_ms / 1000.0;
  const bool backward = c->prm.time_surface_mode == ESVO_TS_BACKWARD;
  const int ks = c->prm.median_blur_kernel_size > 0 ? 2 * c->prm.median_blur_kernel_size + 1 : 1;
  if (ks != 1 && ks != 3) { c->set_error("median_blur_kernel_size > 1 is not supported on the device path"); return ESVO_ERR_UNSUPPORTED; }
  if (backward) {
    if (ks == 3)
      ts_decay_median_kernel<3><<<grd, blk, 0, c->stream>>>(
          s.scalars, (const long long*)s.cur_idx, (const long long*)s.cur_t, s.cur_pol, (const long long*)s.tmp_idx,
          (const long long*)s.tmp_t, s.tmp_pol, s.cnt, c->prm.max_event_queue_len, T, decay_sec, c->prm.ignore_polarity,
          d.W, d.H, d.pitch, (long long*)s.out_idx, s.img_med, maybe_general);
    else
      ts_decay_median_kernel<1><<<grd, blk, 0, c->stream>>>(
          s.scalars, (const long long*)s.cur_idx, (const long long*)s.cur_t, s.cur_pol, (const long long*)s.tmp_idx,
          (const long long*)s.tmp_t, s.tmp_pol, s.cnt, c->prm.max_event_queue_len, T, decay_sec, c->prm.ignore_polarity,
          d.W, d.H, d.pitch, (long long*)s.out_idx, s.img_med, maybe_general);
    dim3 b2(32, 8), g2(div_up(d.W, 32), div_up(d.H, 8));
    ts_remap_kernel<<<g2, b2, 0, c->stream>>>(s.img_med, s.map1, s.map2, d.W, d.H, d.pitch, s.img_out);
    c->launches += 2;
  } else {
    // FORWARD: the splat itself rectifies, no remap afterwards (TimeSurface.cpp:138-142 publishes the image as is)
    if (!s.fwd_lut) {
      ESVO_CUDA_TRY(c, dmalloc(&s.fwd_lut, 2 * npix)); ESVO_CUDA_TRY(c, dmalloc(&s.fwd_head, npix));
      ESVO_CUDA_TRY(c, dmalloc(&s.fwd_next, 4 * npix)); ESVO_CUDA_TRY(c, dmalloc(&s.fwd_val, 4 * npix));
      fill_i32_ts_kernel<<<div_up((int)npix, B), B, 0, c->stream>>>(s.fwd_head, npix, -1);
      c->launches += 1;
    }
    if (s.fwd_tables_version != c->tables_version) {
      ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.fwd_lut, c->cam[cam].lut.data(), 2 * npix * 8, cudaMemcpyHostToDevice, c->stream));
      ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));   // pageable source
      s.fwd_tables_version = c->tables_version;
    }
    ts_forward_scatter_kernel<<<div_up((int)npix, B), B, 0, c->stream>>>(
        s.scalars, (const long long*)s.cur_idx, (const long long*)s.cur_t, s.cur_pol, (const long long*)s.tmp_idx,
        (const long long*)s.tmp_t, s.tmp_pol, s.cnt, c->prm.max_event_queue_len, T, decay_sec, c->prm.ignore_polarity, d.W, d.H,
        s.fwd_lut, (long long*)s.out_idx, s.fwd_head, s.fwd_next, s.fwd_val, maybe_general);
    ts_forward_fold_kernel<<<div_up((int)npix, B), B, 0, c->stream>>>(d.W, d.H, d.pitch, s.fwd_head, s.fwd_next, s.fwd_val,
                                                                     c->prm.ignore_polarity, ks == 3 ? s.img_med : s.img_out);
    c->launches += 2;
    if (ks == 3) {
      dim3 b2(32, 8), g2(div_up(d.W, 32), div_up(d.H, 8));
      ts_median3_kernel<<<g2, b2, 0, c->stream>>>(s.img_med, d.W, d.H, d.pitch, s.img_out);
      c->launches += 1;
    }
  }
  c->prof_end(pe);
  ESVO_CUDA_TRY(c, cudaGetLastError());
  s.built = true;
  s.last_img = s.img_out;
  return ESVO_OK;
}

}  // namespace esvo
