// esvo_b200 product code -- hot pixels of a recorded event stream (sm_90a).
//
// Hot pixels fire whatever the scene does.  The reference leaves them to an offline ROS tool that rewrites the bag (step 4 of
// events_repacking_helper/README.md); here they are counted, selected and dropped on the device, at the packed ingest.
//   count:  per-camera u32 grid c[p], p = y * W + x, over the dvs_msgs/Event wire records with x < W && y < H, accumulated
//           over any number of calls (records outside the image are neither counted nor ever dropped);
//   select: with N = W * H, S1 = sum c, S2 = sum c^2 (exact integers, u64 / u128), each converted once to double (round to
//           nearest): mu = S1 / N, sigma = sqrt(max(0, S2 / N - mu * mu)), p is hot iff (double)c[p] > mu + k * sigma, in
//           IEEE double in this order without contraction (numpy reproduces every decision);
//   drop:   while a mask is installed, ts_push_packed first copies the records whose in-image pixel is not hot, in order, into
//           a buffer of the camera (three passes, as events.cu's ordered compaction), and pushes those.
#include <cmath>

#include "common.cuh"

namespace esvo {

__device__ int block_excl_scan(int v, int* s_warp, int& total);   // bm.cu

// TsState::HotPix::d_scal
enum { HP_OVERFLOW = 0, HP_S1, HP_S2_LO, HP_S2_HI, HP_NHOT, HP_THR, HP_KEPT, HP_LAST_T, HP_NSCAL };
constexpr int kHpBlock = 256;   // 8 warps: one packed_stage_warp stage each

// ---- count: one warp per 32 records.  Hot pixels are exactly the contended bins, so the lanes of a warp that share a pixel
// add together: the lowest of them adds the group's size.  A count that would pass 2^32 - 1 raises the overflow flag (the
// selection then refuses the counts).
__global__ void __launch_bounds__(kHpBlock) hp_count_packed_kernel(const uint8_t* __restrict__ src, size_t n, int W, int H,
                                                                   uint32_t* __restrict__ counts, unsigned long long* __restrict__ scal) {
  __shared__ uint32_t stage[kHpBlock / 32][kPackWords];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t i0 = blockIdx.x * (size_t)blockDim.x + (size_t)w * 32;
  if (i0 >= n) return;   // uniform per warp
  const size_t i = i0 + lane;
  const uint8_t* r = packed_stage_warp(src, n, i0, lane, stage[w]);
  int p = -1;
  if (i < n) {
    const int x = packed_x(r), y = packed_y(r);
    if (x < W && y < H) p = y * W + x;
  }
  const unsigned peers = __match_any_sync(0xffffffffu, p);
  if (p >= 0 && lane == __ffs(peers) - 1) {
    const unsigned add = (unsigned)__popc(peers);
    const unsigned old = atomicAdd(&counts[p], add);
    if (old > 0xffffffffu - add) scal[HP_OVERFLOW] = 1;
  }
}

// ---- select, (1): S1 and S2 over the grid.  Integer sums do not depend on the order, so each warp adds its partial sums
// atomically; S2 is 128-bit, its low word's carries go to the high word.
__global__ void __launch_bounds__(256) hp_sums_kernel(const uint32_t* __restrict__ counts, size_t npix, unsigned long long* scal) {
  unsigned long long s1 = 0;
  unsigned __int128 s2 = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long v = counts[i];
    s1 += v;
    s2 += v * v;                                  // < 2^64 for v < 2^32
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    const unsigned long long lo = __shfl_xor_sync(0xffffffffu, (unsigned long long)s2, o);
    const unsigned long long hi = __shfl_xor_sync(0xffffffffu, (unsigned long long)(s2 >> 64), o);
    s2 += ((unsigned __int128)hi << 64) | lo;
  }
  if ((threadIdx.x & 31) == 0 && s1) {
    const unsigned long long lo = (unsigned long long)s2, hi = (unsigned long long)(s2 >> 64);
    atomicAdd(&scal[HP_S1], s1);
    const unsigned long long old = atomicAdd(&scal[HP_S2_LO], lo);
    atomicAdd(&scal[HP_S2_HI], hi + (old + lo < old ? 1ull : 0ull));
  }
}
// a 128-bit unsigned integer to the nearest double (ties to even): the top 64 bits, with every lower bit folded into a sticky
// bit below the rounding position, rounded once, then scaled by an exact power of two
__device__ __forceinline__ double u128_to_double_rn(unsigned long long hi, unsigned long long lo) {
  if (hi == 0) return __ull2double_rn(lo);
  const int s = __clzll((long long)hi);
  const unsigned long long top = s ? (hi << s) | (lo >> (64 - s)) : hi;
  const unsigned long long rest = s ? lo << s : lo;
  return ldexp(__ull2double_rn(top | (rest != 0 ? 1ull : 0ull)), 64 - s);
}
// (2): the threshold, once
__global__ void hp_threshold_kernel(unsigned long long* scal, size_t npix, double k) {
  if (threadIdx.x || blockIdx.x) return;
  const double N = (double)npix;
  const double mu = __ddiv_rn(__ull2double_rn(scal[HP_S1]), N);
  const double s2 = u128_to_double_rn(scal[HP_S2_HI], scal[HP_S2_LO]);
  const double var = __dsub_rn(__ddiv_rn(s2, N), __dmul_rn(mu, mu));
  const double sigma = __dsqrt_rn(var > 0.0 ? var : 0.0);
  const double thr = __dadd_rn(mu, __dmul_rn(k, sigma));
  scal[HP_THR] = (unsigned long long)__double_as_longlong(thr);
}
// (3): the mask and the number of hot pixels.  Overflowed counts leave the mask as it was.
__global__ void __launch_bounds__(256) hp_mask_kernel(const uint32_t* __restrict__ counts, size_t npix, unsigned long long* scal,
                                                      uint8_t* __restrict__ mask) {
  if (scal[HP_OVERFLOW]) return;
  const double thr = __longlong_as_double((long long)scal[HP_THR]);
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const bool hot = i < npix && (double)counts[i] > thr;
  if (i < npix) mask[i] = hot ? 1 : 0;
  const unsigned b = __ballot_sync(0xffffffffu, hot);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(&scal[HP_NHOT], (unsigned long long)__popc(b));
}

// ---- masked ingest: ordered compaction of the records whose in-image pixel is not hot.  (1) every block of 256 records counts
// its kept ones, (2) one block turns the counts into exclusive offsets and publishes the number kept, (3) every block scans its
// own flags from its offset, copies its kept records and the last kept one publishes its stamp.
__device__ __forceinline__ int hp_keep(const uint8_t* r, const uint8_t* __restrict__ mask, int W, int H) {
  const int x = packed_x(r), y = packed_y(r);
  return !(x < W && y < H && mask[(size_t)y * W + x]);
}
__global__ void __launch_bounds__(kHpBlock) hp_compact_count_kernel(const uint8_t* __restrict__ src, size_t n, int W, int H,
                                                                    const uint8_t* __restrict__ mask, int* __restrict__ blk) {
  __shared__ uint32_t stage[kHpBlock / 32][kPackWords];
  __shared__ int s_warp[33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t i0 = blockIdx.x * (size_t)blockDim.x + (size_t)w * 32, i = i0 + lane;
  const uint8_t* r = packed_stage_warp(src, n, i0, lane, stage[w]);
  const int f = i < n ? hp_keep(r, mask, W, H) : 0;
  int total;
  block_excl_scan(f, s_warp, total);
  if (threadIdx.x == 0) blk[blockIdx.x] = total;
}
__global__ void __launch_bounds__(1024) hp_compact_offsets_kernel(int* __restrict__ blk, int nb, unsigned long long* __restrict__ scal) {
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
  if (threadIdx.x == 0) scal[HP_KEPT] = (unsigned long long)carry;
}
__global__ void __launch_bounds__(kHpBlock) hp_compact_kernel(const uint8_t* __restrict__ src, size_t n, int W, int H,
                                                              const uint8_t* __restrict__ mask, const int* __restrict__ blk,
                                                              unsigned long long* __restrict__ scal, uint8_t* __restrict__ dst) {
  __shared__ uint32_t stage[kHpBlock / 32][kPackWords];
  __shared__ int s_warp[33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t i0 = blockIdx.x * (size_t)blockDim.x + (size_t)w * 32, i = i0 + lane;
  const uint8_t* r = packed_stage_warp(src, n, i0, lane, stage[w]);
  const int f = i < n ? hp_keep(r, mask, W, H) : 0;
  int total;
  const int local = block_excl_scan(f, s_warp, total);
  if (!f) return;
  const unsigned long long pos = (unsigned long long)blk[blockIdx.x] + local;
  uint8_t* d = dst + pos * kPackRec;
#pragma unroll
  for (int q = 0; q < kPackRec; ++q) d[q] = r[q];
  if (pos + 1 == scal[HP_KEPT]) scal[HP_LAST_T] = (unsigned long long)packed_stamp(r);
}

// --------------------------------------------------------------------------------------------

int hp_alloc(Ctx* c, int cam) {
  TsState::HotPix& h = c->ts[cam].hp;
  if (h.counts) return ESVO_OK;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  ESVO_CUDA_TRY(c, dmalloc(&h.counts, npix)); ESVO_CUDA_TRY(c, dmalloc(&h.mask, npix)); ESVO_CUDA_TRY(c, dmalloc(&h.d_scal, HP_NSCAL));
  ESVO_CUDA_TRY(c, cudaMallocHost((void**)&h.h_scal, HP_NSCAL * sizeof(unsigned long long)));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.counts, 0, npix * sizeof(uint32_t), c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.mask, 0, npix, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.d_scal, 0, HP_NSCAL * sizeof(unsigned long long), c->stream));
  return ESVO_OK;
}
void hp_free(TsState& s) {
  TsState::HotPix& h = s.hp;
  void* ps[] = {h.counts, h.mask, h.kept, h.blk, h.d_scal};
  for (void* p : ps) if (p) cudaFree(p);
  if (h.h_scal) cudaFreeHost(h.h_scal);
  h = TsState::HotPix();
}

int hp_count_packed(Ctx* c, int cam, const uint8_t* src, size_t n) {
  int rc = hp_alloc(c, cam);
  if (rc || n == 0) return rc;
  TsState::HotPix& h = c->ts[cam].hp;
  hp_count_packed_kernel<<<(unsigned)((n + kHpBlock - 1) / kHpBlock), kHpBlock, 0, c->stream>>>(src, n, c->dc.W, c->dc.H, h.counts, h.d_scal);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

// Host runs go through the camera's pinned staging block (ts_pack_staging), at most kCountChunk records per copy: a whole
// recording is counted in pieces of one staging fill each.
int hp_count_packed_host(Ctx* c, int cam, const uint8_t* const* runs, const size_t* n_events, int n_runs) {
  constexpr size_t kCountChunk = (size_t)1 << 20;
  TsState& s = c->ts[cam];
  size_t n = 0;
  for (int k = 0; k < n_runs; ++k) n += n_events[k];
  int rc = hp_alloc(c, cam);
  if (rc || n == 0) return rc;
  const size_t chunk = std::min(n, kCountChunk);
  if ((rc = ts_pack_staging(c, cam, chunk * kPackRec))) return rc;
  size_t fill = 0;
  auto flush = [&]() -> int {
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(s.pack_dev, s.h_pack, fill * kPackRec, cudaMemcpyHostToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaEventRecord(s.ev_pack, c->stream));
    int r = hp_count_packed(c, cam, s.pack_dev, fill);
    fill = 0;
    return r ? r : ts_pack_staging(c, cam, chunk * kPackRec);   // waits for the copy before the block is refilled
  };
  for (int k = 0; k < n_runs; ++k) {
    for (size_t done = 0; done < n_events[k];) {
      const size_t m = std::min(n_events[k] - done, chunk - fill);
      std::memcpy(s.h_pack + fill * kPackRec, runs[k] + done * kPackRec, m * kPackRec);
      fill += m; done += m;
      if (fill == chunk && (rc = flush())) return rc;
    }
  }
  return fill ? flush() : ESVO_OK;
}

int hp_select(Ctx* c, int cam, double k, int64_t* n_hot) {
  if (!(k >= 0.0) || !std::isfinite(k)) { c->set_error("esvo_hotpix_select: k must be finite and >= 0"); return ESVO_ERR_INVALID_ARG; }
  int rc = hp_alloc(c, cam);
  if (rc) return rc;
  TsState::HotPix& h = c->ts[cam].hp;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.d_scal + HP_S1, 0, (HP_NHOT - HP_S1 + 1) * sizeof(unsigned long long), c->stream));
  hp_sums_kernel<<<c->num_sms * 4, 256, 0, c->stream>>>(h.counts, npix, h.d_scal);
  hp_threshold_kernel<<<1, 32, 0, c->stream>>>(h.d_scal, npix, k);
  hp_mask_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, c->stream>>>(h.counts, npix, h.d_scal, h.mask);
  c->launches += 3;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h.h_scal, h.d_scal, HP_NSCAL * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (h.h_scal[HP_OVERFLOW]) {
    c->set_error("esvo_hotpix_select: a pixel was counted more than 2^32 - 1 times; the counts are refused (esvo_hotpix_clear)");
    return ESVO_ERR_CAPACITY;
  }
  h.masked = h.h_scal[HP_NHOT] > 0;   // a mask without a hot pixel filters nothing: the pushes stay unfiltered (no read-back)
  if (n_hot) *n_hot = (int64_t)h.h_scal[HP_NHOT];
  return ESVO_OK;
}

int hp_read(Ctx* c, int cam, uint32_t* counts, uint8_t* mask) {
  int rc = hp_alloc(c, cam);
  if (rc) return rc;
  TsState::HotPix& h = c->ts[cam].hp;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  if (counts) ESVO_CUDA_TRY(c, cudaMemcpyAsync(counts, h.counts, npix * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
  if (mask) ESVO_CUDA_TRY(c, cudaMemcpyAsync(mask, h.mask, npix, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  return ESVO_OK;
}

int hp_clear(Ctx* c, int cam) {
  int rc = hp_alloc(c, cam);
  if (rc) return rc;
  TsState::HotPix& h = c->ts[cam].hp;
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.counts, 0, npix * sizeof(uint32_t), c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.mask, 0, npix, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(h.d_scal, 0, HP_NSCAL * sizeof(unsigned long long), c->stream));
  h.masked = false;
  return ESVO_OK;
}

// n records at src (device) -> the kept ones at *kept (this camera's buffer, valid until its next masked push), their number
// and the last one's stamp.  One read-back: the caller needs both on the host.
int hp_compact_packed(Ctx* c, int cam, const uint8_t* src, size_t n, const uint8_t** kept, size_t* n_kept, int64_t* last_t) {
  TsState::HotPix& h = c->ts[cam].hp;
  const size_t bytes = n * kPackRec, nb = (n + kHpBlock - 1) / kHpBlock;
  if (bytes > h.kept_cap || nb > h.blk_cap) {
    ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (bytes > h.kept_cap) {
      if (h.kept) cudaFree(h.kept);
      h.kept = nullptr;
      h.kept_cap = std::max<size_t>(2 * bytes, (size_t)1 << 20);
      ESVO_CUDA_TRY(c, dmalloc(&h.kept, h.kept_cap));
    }
    if (nb > h.blk_cap) {
      if (h.blk) cudaFree(h.blk);
      h.blk = nullptr;
      h.blk_cap = std::max<size_t>(2 * nb, 1024);
      ESVO_CUDA_TRY(c, dmalloc(&h.blk, h.blk_cap));
    }
  }
  const int W = c->dc.W, H = c->dc.H;
  hp_compact_count_kernel<<<(unsigned)nb, kHpBlock, 0, c->stream>>>(src, n, W, H, h.mask, h.blk);
  hp_compact_offsets_kernel<<<1, 1024, 0, c->stream>>>(h.blk, (int)nb, h.d_scal);
  hp_compact_kernel<<<(unsigned)nb, kHpBlock, 0, c->stream>>>(src, n, W, H, h.mask, h.blk, h.d_scal, h.kept);
  c->launches += 3;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h.h_scal + HP_KEPT, h.d_scal + HP_KEPT, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  *kept = h.kept;
  *n_kept = (size_t)h.h_scal[HP_KEPT];
  *last_t = (int64_t)h.h_scal[HP_LAST_T];
  return ESVO_OK;
}

}  // namespace esvo
