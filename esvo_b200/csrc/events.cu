// esvo_b200 product code -- event windows read from the resident time-surface log (sm_90a).
//
// Replaces the host event buffers the closed loop's nodes keep only to search them:
//   * tools::EventBuffer_lower_bound (utils.h:50-55) over esvo_Tracking's events_left_ (curDataTransferring,
//     esvo_Tracking.cpp:240-263);
//   * the newest-first walks of esvo_Mapping::dataTransferring (esvo_Mapping.cpp:538-552 SGM, :554-575 BM) over the
//     mapper's events_left_;
//   * createDenoisingMask + extractDenoisedEvents (esvo_Mapping.cpp:282-296,1046-1072).
// The nodes' deques hold every left event they were handed, insertion-sorted and capped (mapper 3e6, tracker 5e6, the
// tracker's cleared by its reset()).  Camera 0's log (ts.cu) holds the same events in push order, so for ordered input a
// deque is the logical buffer [front, total) of global push indices, front = where the deque would begin.  The log keeps
// at least its newest log_cap / 4 events resident; what the answer needs must lie there (or be pinned by the two stamps the
// fold records), otherwise the call is refused.
#include <algorithm>

#include "common.cuh"

namespace esvo {

__device__ int block_excl_scan(int v, int* s_warp, int& total);                                  // bm.cu
__global__ void ts_median3_kernel(const uint8_t* __restrict__ src, int W, int H, int pitch, uint8_t* __restrict__ dst);   // ts.cu

// Scalars of one window (Ctx::EventWindow::d_scal): status, events walked, local index of the first (newest) walked event,
// events kept, lower_bound(t_end), lower_bound(t_begin) (global; -1 when not determined).
enum { EW_STATUS = 0, EW_WALKED, EW_START, EW_KEPT, EW_END, EW_BEGIN, EW_NSCAL = 8 };
enum { EW_OK = 0, EW_FOLDED = 1, EW_UNORDERED = 2 };

// What the resident log knows about the events before it: the newest folded stamp (scalars[10..11], written by the fold) and
// the stamp of the very first event pushed (scalars[12..13], kept by the first fold).  Every folded event lies between them.
struct FoldInfo { long long base, n; double t_fold, t_first; };
__device__ __forceinline__ FoldInfo fold_info(const int32_t* __restrict__ scal, long long log_base, long long log_n) {
  long long tf, t0;
  memcpy(&tf, scal + 10, 8); memcpy(&t0, scal + 12, 8);
  return FoldInfo{log_base, log_n, ns_to_sec_dev(tf), ns_to_sec_dev(t0)};
}
// tools::EventBuffer_lower_bound over [front, base + n): the first index whose toSec() is not below v (toSec() doubles, so
// stamps that share a double are equal; ns_to_sec_dev rounds the product and the sum separately, as the host does).
// known = false when the answer lies among the folded events and is not pinned by their stamp range.
__device__ __forceinline__ long long lower_bound_log(const int64_t* __restrict__ et, const FoldInfo& f, long long front, double v,
                                                     bool& known) {
  long long lo = max(front, f.base) - f.base, hi = f.n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (ns_to_sec_dev(et[mid]) < v) lo = mid + 1; else hi = mid;
  }
  known = true;
  if (front < f.base && lo == 0) {             // every resident event is >= v: the bound is in [front, base]
    if (f.t_fold < v) return f.base;           // every folded event is < v
    if (v <= f.t_first) return front;          // every event is >= v
    known = false;
  }
  return f.base + lo;
}

// One thread: the two bounds, the one-past-the-end rule and the walk's extent (frontend::selectCloseEvents /
// selectSGMEvents).  budget: PROCESS_EVENT_NUM for BM, PROCESS_EVENT_NUM + 1 for SGM.
__global__ void ew_bounds_kernel(const int64_t* __restrict__ et, const int32_t* __restrict__ scal, long long log_base, long long log_n,
                                 long long front, double t_begin, double t_end, long long budget, long long* __restrict__ out) {
  if (threadIdx.x || blockIdx.x) return;
  for (int k = 0; k < EW_NSCAL; ++k) out[k] = 0;
  out[EW_END] = out[EW_BEGIN] = -1;
  if (scal[1]) { out[EW_STATUS] = EW_UNORDERED; return; }
  const FoldInfo f = fold_info(scal, log_base, log_n);
  const long long total = log_base + log_n;
  bool known_end, known_begin;
  long long e_end = lower_bound_log(et, f, front, t_end, known_end);
  const long long e_begin = lower_bound_log(et, f, front, t_begin, known_begin);
  if (!known_end) { out[EW_STATUS] = EW_FOLDED; return; }
  out[EW_END] = e_end;
  if (known_begin) out[EW_BEGIN] = e_begin;
  // no event at or after t_end: the reference's first push is the slot one past the newest event; it is skipped but keeps its
  // place in the budget
  if (e_end == total && (!known_begin || e_end != e_begin) && budget > 0) { --e_end; --budget; }
  // an undetermined lower_bound(t_begin) lies below the resident log, so only the budget can end the walk inside it
  const long long n = known_begin ? (e_end > e_begin ? min(budget, e_end - e_begin) : 0) : budget;
  if (n > 0 && e_end - n + 1 < log_base) { out[EW_STATUS] = EW_FOLDED; return; }   // the walk would leave the resident log
  out[EW_WALKED] = n;
  out[EW_START] = e_end - log_base;
}

// The walk: walked event i is log[start - i].  With denoising, also Visualization::plot_eventMap of the walked events
// (Visualization.cpp:96-104: only x < W && y < H) into the zeroed event map.
__global__ void ew_walk_kernel(const uint16_t* __restrict__ ex, const uint16_t* __restrict__ ey, const int64_t* __restrict__ et,
                               const long long* __restrict__ scal, int cap, int W, int H, uint16_t* __restrict__ wx,
                               uint16_t* __restrict__ wy, int64_t* __restrict__ wt, uint8_t* __restrict__ evmap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap || scal[EW_STATUS] != EW_OK || i >= scal[EW_WALKED]) return;
  const long long j = scal[EW_START] - i;
  const int x = ex[j], y = ey[j];
  wx[i] = (uint16_t)x; wy[i] = (uint16_t)y; wt[i] = et[j];
  if (evmap && x < W && y < H) evmap[(size_t)y * W + x] = 255;
}

// Ordered compaction of the walked events (extractDenoisedEvents, esvo_Mapping.cpp:1062-1072): keep event i when the mask is
// 255 at the flat index y * W + x -- cv::Mat::at<uchar>(y, x) on a continuous image, so x == W reads the first pixel of row
// y + 1 -- in walk order, at most max_keep.  A flat index past the image reads outside the reference's buffer (undefined);
// such an event is not kept here.  mask == nullptr: every walked event is a candidate (no denoising).
// Three passes, linear in the walk: (1) every block of 256 positions counts its kept events, (2) one block turns the counts into
// exclusive offsets and publishes the number kept, (3) every block scans its own flags from its offset and scatters.
constexpr int kEwBlock = 256;
__device__ __forceinline__ int ew_keep(const uint16_t* __restrict__ wx, const uint16_t* __restrict__ wy, const uint8_t* __restrict__ mask,
                                       int W, int H, int n, int i) {
  if (i >= n) return 0;
  if (!mask) return 1;
  const size_t p = (size_t)wy[i] * W + wx[i];
  return p < (size_t)W * H && mask[p] == 255;
}
__device__ __forceinline__ int ew_walked(const long long* __restrict__ scal) {
  return scal[EW_STATUS] == EW_OK ? (int)scal[EW_WALKED] : 0;
}
__global__ void __launch_bounds__(kEwBlock) ew_count_kernel(const uint16_t* __restrict__ wx, const uint16_t* __restrict__ wy,
                                                            const uint8_t* __restrict__ mask, int W, int H, const long long* __restrict__ scal,
                                                            int* __restrict__ blk) {
  __shared__ int s_warp[33];
  const int f = ew_keep(wx, wy, mask, W, H, ew_walked(scal), blockIdx.x * kEwBlock + threadIdx.x);
  int total;
  block_excl_scan(f, s_warp, total);
  if (threadIdx.x == 0) blk[blockIdx.x] = total;
}
__global__ void __launch_bounds__(1024) ew_offsets_kernel(int* __restrict__ blk, int nb, long long max_keep, long long* __restrict__ scal) {
  __shared__ int s_warp[33];
  int carry = 0;
  for (int b0 = 0; b0 < nb; b0 += 1024) {
    const int b = b0 + threadIdx.x;
    const int v = b < nb ? blk[b] : 0;
    int total;
    const int ex = block_excl_scan(v, s_warp, total);   // ends with a barrier: every read of this chunk is done
    if (b < nb) blk[b] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) scal[EW_KEPT] = min((long long)carry, max_keep);
}
__global__ void __launch_bounds__(kEwBlock) ew_compact_kernel(const uint16_t* __restrict__ wx, const uint16_t* __restrict__ wy,
                                                              const int64_t* __restrict__ wt, const uint8_t* __restrict__ mask, int W, int H,
                                                              long long max_keep, const long long* __restrict__ scal, const int* __restrict__ blk,
                                                              uint16_t* __restrict__ kx, uint16_t* __restrict__ ky, int64_t* __restrict__ kt) {
  __shared__ int s_warp[33];
  const int n = ew_walked(scal);
  if (blockIdx.x * kEwBlock >= n) return;              // uniform per block
  const int i = blockIdx.x * kEwBlock + threadIdx.x;
  const int f = ew_keep(wx, wy, mask, W, H, n, i);
  int total;
  const int local = block_excl_scan(f, s_warp, total);
  const long long pos = (long long)blk[blockIdx.x] + local;
  if (f && pos < max_keep) { kx[pos] = wx[i]; ky[pos] = wy[i]; kt[pos] = wt[i]; }
}

// k lower bounds at once (esvo_events_lower_bound_dev); out[q] = -1 when not determined by what the log knows
__global__ void ew_lower_bounds_kernel(const int64_t* __restrict__ et, const int32_t* __restrict__ scal, long long log_base, long long log_n,
                                       long long front, const long long* __restrict__ q, int k, long long* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  if (scal[1]) { out[i] = -2; return; }
  const FoldInfo f = fold_info(scal, log_base, log_n);
  bool known;
  const long long r = lower_bound_log(et, f, front, ns_to_sec_dev(q[i]), known);
  out[i] = known ? r : -1;
}

// --------------------------------------------------------------------------------------------

static int ew_alloc(Ctx* c, size_t cap) {
  Ctx::EventWindow& w = c->evw;
  if (!w.d_scal) {
    const size_t npix = (size_t)c->dc.W * c->dc.H;
    ESVO_CUDA_TRY(c, dmalloc(&w.d_scal, EW_NSCAL + 2 * Ctx::EventWindow::kMaxQueries));
    ESVO_CUDA_TRY(c, cudaMallocHost((void**)&w.h_scal, (EW_NSCAL + 2 * Ctx::EventWindow::kMaxQueries) * sizeof(long long)));
    ESVO_CUDA_TRY(c, dmalloc(&w.evmap, npix)); ESVO_CUDA_TRY(c, dmalloc(&w.mask, npix));
  }
  if (cap > w.cap) {
    ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));   // the previous selection may still be read by a frame
    void* olds[] = {w.wx, w.wy, w.wt, w.kx, w.ky, w.kt, w.blk};
    for (void* p : olds) if (p) cudaFree(p);
    w.cap = std::max<size_t>(cap, 1024);
    ESVO_CUDA_TRY(c, dmalloc(&w.wx, w.cap)); ESVO_CUDA_TRY(c, dmalloc(&w.wy, w.cap)); ESVO_CUDA_TRY(c, dmalloc(&w.wt, w.cap));
    ESVO_CUDA_TRY(c, dmalloc(&w.kx, w.cap)); ESVO_CUDA_TRY(c, dmalloc(&w.ky, w.cap)); ESVO_CUDA_TRY(c, dmalloc(&w.kt, w.cap));
    ESVO_CUDA_TRY(c, dmalloc(&w.blk, (size_t)div_up((int)w.cap, kEwBlock)));
  }
  return ESVO_OK;
}
void ew_free(Ctx* c) {
  Ctx::EventWindow& w = c->evw;
  void* ps[] = {w.wx, w.wy, w.wt, w.kx, w.ky, w.kt, w.blk, w.evmap, w.mask, w.d_scal};
  for (void* p : ps) if (p) cudaFree(p);
  if (w.h_scal) cudaFreeHost(w.h_scal);
  w = Ctx::EventWindow();
}

static int ew_check(Ctx* c, int cam, int64_t front, const char* who) {
  const TsState& s = c->ts[cam];
  if (c->depth > 1) { c->set_error(std::string(who) + ": not available at pipeline depth > 1"); return ESVO_ERR_STATE; }
  if (s.unordered) {
    c->set_error(std::string(who) + ": the camera takes unordered input; the log is in arrival order, the nodes' buffers are sorted");
    return ESVO_ERR_UNSUPPORTED;
  }
  if (front < 0 || front > s.log_base + (int64_t)s.log_n) {
    c->set_error(std::string(who) + ": front " + std::to_string((long long)front) + " is outside [0, " +
                 std::to_string((long long)(s.log_base + (int64_t)s.log_n)) + "]");
    return ESVO_ERR_INVALID_ARG;
  }
  return ESVO_OK;
}

int events_window(Ctx* c, int cam, int64_t front, int64_t t_begin_ns, int64_t t_end_ns, size_t budget, int denoise, size_t max_keep,
                  size_t* n_out) {
  static const char* who = "esvo_events_window_dev";
  int rc = ew_check(c, cam, front, who);
  if (rc) return rc;
  if (t_begin_ns > t_end_ns) { c->set_error(std::string(who) + ": t_begin_ns > t_end_ns"); return ESVO_ERR_INVALID_ARG; }
  Ctx::EventWindow& w = c->evw;
  w.valid = false;
  const TsState& s = c->ts[cam];
  const size_t cap = std::min(budget, s.log_n);           // the walk never leaves the resident log
  if ((rc = ew_alloc(c, std::max<size_t>(cap, 1)))) return rc;   // the compaction writes one block count even for an empty walk
  const DevConsts& d = c->dc;
  const size_t npix = (size_t)d.W * d.H;
  auto sec = [](int64_t ns) { int64_t q = ns / 1000000000LL, r = ns % 1000000000LL; if (r < 0) { r += 1000000000LL; --q; } return (double)q + 1e-9 * (double)r; };
  ew_bounds_kernel<<<1, 32, 0, c->stream>>>(s.et, s.scalars, s.log_base, (long long)s.log_n, front, sec(t_begin_ns), sec(t_end_ns),
                                            (long long)std::min<size_t>(budget, (size_t)INT64_MAX), w.d_scal);
  c->launches += 1;
  if (denoise) ESVO_CUDA_TRY(c, cudaMemsetAsync(w.evmap, 0, npix, c->stream));
  const int B = 256;
  if (cap) {
    ew_walk_kernel<<<div_up((int)cap, B), B, 0, c->stream>>>(s.ex, s.ey, s.et, w.d_scal, (int)cap, d.W, d.H, w.wx, w.wy, w.wt,
                                                            denoise ? w.evmap : nullptr);
    c->launches += 1;
  }
  if (denoise) {                               // cv::medianBlur 3x3 on the 0/255 map: 255 iff at least 5 of the 9 are on
    dim3 b2(32, 8), g2(div_up(d.W, 32), div_up(d.H, 8));
    ts_median3_kernel<<<g2, b2, 0, c->stream>>>(w.evmap, d.W, d.H, d.W, w.mask);
    c->launches += 1;
  }
  const int nb = std::max(1, div_up((int)cap, kEwBlock));
  const uint8_t* m = denoise ? w.mask : nullptr;
  const long long keep_max = (long long)std::min<size_t>(max_keep, (size_t)INT64_MAX);
  ew_count_kernel<<<nb, kEwBlock, 0, c->stream>>>(w.wx, w.wy, m, d.W, d.H, w.d_scal, w.blk);
  ew_offsets_kernel<<<1, 1024, 0, c->stream>>>(w.blk, nb, keep_max, w.d_scal);
  ew_compact_kernel<<<nb, kEwBlock, 0, c->stream>>>(w.wx, w.wy, w.wt, m, d.W, d.H, keep_max, w.d_scal, w.blk, w.kx, w.ky, w.kt);
  c->launches += 3;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(w.h_scal, w.d_scal, EW_NSCAL * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  const long long* h = w.h_scal;
  if (h[EW_STATUS] == EW_UNORDERED) {
    c->set_error(std::string(who) + ": events were not pushed in time order");
    return ESVO_ERR_UNSUPPORTED;
  }
  if (h[EW_STATUS] == EW_FOLDED) {
    c->set_error(std::string(who) + ": the window reaches events folded out of the resident log (the newest " +
                 std::to_string(s.log_n) + " of " + std::to_string((long long)(s.log_base + (int64_t)s.log_n)) + " are resident)");
    return ESVO_ERR_UNSUPPORTED;
  }
  w.n = (size_t)h[EW_KEPT]; w.walked = (size_t)h[EW_WALKED];
  w.valid = true;
  if (n_out) *n_out = w.n;
  return ESVO_OK;
}

int events_lower_bound(Ctx* c, int cam, int64_t front, const int64_t* t_ns, size_t k, int64_t* idx_out) {
  static const char* who = "esvo_events_lower_bound_dev";
  int rc = ew_check(c, cam, front, who);
  if (rc) return rc;
  if (k > (size_t)Ctx::EventWindow::kMaxQueries) { c->set_error(std::string(who) + ": more than 64 stamps"); return ESVO_ERR_INVALID_ARG; }
  if (k == 0) return ESVO_OK;
  if ((rc = ew_alloc(c, 0))) return rc;
  Ctx::EventWindow& w = c->evw;
  const TsState& s = c->ts[cam];
  long long* hq = w.h_scal + EW_NSCAL;
  long long* dq = w.d_scal + EW_NSCAL;
  for (size_t i = 0; i < k; ++i) hq[i] = t_ns[i];
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(dq, hq, k * sizeof(long long), cudaMemcpyHostToDevice, c->stream));
  ew_lower_bounds_kernel<<<1, Ctx::EventWindow::kMaxQueries, 0, c->stream>>>(s.et, s.scalars, s.log_base, (long long)s.log_n, front, dq, (int)k,
                                                                        dq + Ctx::EventWindow::kMaxQueries);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  long long* hr = hq + Ctx::EventWindow::kMaxQueries;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(hr, dq + Ctx::EventWindow::kMaxQueries, k * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  for (size_t i = 0; i < k; ++i)
    if (hr[i] == -2) { c->set_error(std::string(who) + ": events were not pushed in time order"); return ESVO_ERR_UNSUPPORTED; }
  // every bound the log determines is written; one it does not is -1, and the call is refused
  int rc_out = ESVO_OK;
  for (size_t i = 0; i < k; ++i) {
    idx_out[i] = hr[i];
    if (hr[i] == -1 && rc_out == ESVO_OK) {
      c->set_error(std::string(who) + ": the bound of stamp " + std::to_string((long long)t_ns[i]) + " lies among events folded out of the resident log");
      rc_out = ESVO_ERR_UNSUPPORTED;
    }
  }
  return rc_out;
}

}  // namespace esvo
