// esvo_b200 product code -- the chunk inflater of compressed ROS bags (include/esvo_b200_inflate.h), sm_90a.
//
// A call packs the chunks into batches that fit the scratch.  Scratch layout of a batch:
//   [Desc per chunk | bz2 chunk list | LZ4 chunk list] [compressed inputs] [outputs] [bz2 work regions]
// The first two parts go up in one copy from pinned staging; the descriptors (with each chunk's refusal) and the outputs
// come back in two.  The kernels are the stages of inflate_core.h:
//   bz2_parse_kernel        one warp per chunk (lane 0 decodes; the symbol decode is serial per block), state in shared;
//   bz2_hist_kernel         one thread per tile of kTile positions: its 256 counters in a shared column;
//   bz2_scan_kernel         one CUDA block per bz2 block, one thread per symbol: the scan over tiles, then over symbols;
//   bz2_scatter_kernel      one thread per tile: tt[pos[L[i]]++] |= i << 8;
//   bz2_walk_len_kernel     one thread per sample: walk to the next sample;
//   bz2_order_kernel        one thread per block: chain the segments;
//   bz2_walk_write_kernel   one thread per sample: walk again, writing the bytes;
//   bz2_unrle_count_kernel  one thread per block: decoded length and CRC;
//   bz2_finish_kernel       one thread per chunk: CRCs, offsets, size;
//   bz2_unrle_write_kernel  one thread per block: decoded bytes;
//   lz4_frame_kernel        one warp per frame.
// Every stage skips a chunk that an earlier stage refused.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/esvo_b200_inflate.h"
#include "inflate_core.h"

// The kernels and helpers live in a named namespace (not an anonymous one), so each kernel keeps one stable symbol,
// esvo_inflate::bz2_*_kernel / lz4_frame_kernel, that a profiler trace can attribute time to.
namespace esvo_inflate {

constexpr size_t kAlign = 256;
size_t alignUp(size_t v) { return (v + kAlign - 1) / kAlign * kAlign; }

// A bz2 chunk's work region, from its caps
struct Layout {
  size_t blk, tt, pre, hist, slen, ssucc, soff, bytes;
  __host__ __device__ explicit Layout(const Bz2Caps& c) {
    size_t o = 0;
    auto take = [&](size_t b) { const size_t r = o; o += (b + 255) / 256 * 256; return r; };
    blk = take(sizeof(Bz2Block) * c.nb);
    tt = take(4ull * c.tt);
    pre = take(c.tt);
    hist = take(1024ull * c.tiles);
    slen = take(4ull * c.samp);
    ssucc = take(4ull * c.samp);
    soff = take(4ull * c.samp);
    bytes = o;
  }
};

struct Desc {
  uint64_t src, src_size, dst, dst_size, work;   // byte offsets in the scratch
  int32_t codec, reason;
  uint32_t nb, comb;
};

struct Batch {
  uint8_t* base;
  Desc* desc;
  const uint32_t* bz;   // the bz2 chunks' indices
  const uint32_t* lz;   // the LZ4 chunks' indices
};

struct Bz2View {   // one bz2 chunk's arrays
  Desc* d;
  Bz2Block* blk;
  uint32_t *tt, *hist, *slen, *ssucc, *soff;
  uint8_t* pre;
  __device__ Bz2View(const Batch& b, uint32_t k) {
    d = &b.desc[b.bz[k]];
    const Layout L(bz2Caps(d->dst_size));
    uint8_t* w = b.base + d->work;
    blk = (Bz2Block*)(w + L.blk); tt = (uint32_t*)(w + L.tt); pre = w + L.pre; hist = (uint32_t*)(w + L.hist);
    slen = (uint32_t*)(w + L.slen); ssucc = (uint32_t*)(w + L.ssucc); soff = (uint32_t*)(w + L.soff);
  }
  // the block holding item i of a per-block numbering (tile0 / samp0 ascending); nb when i is past the last block's items
  __device__ uint32_t find(uint32_t i, bool samples) const {
    const uint32_t nb = d->nb;
    if (nb == 0) return 0;
    const Bz2Block& last = blk[nb - 1];
    if (i >= (samples ? last.samp0 + last.nsamp : last.tile0 + last.ntiles)) return nb;
    uint32_t lo = 0, hi = nb - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) / 2;
      if ((samples ? blk[mid].samp0 : blk[mid].tile0) <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
  }
};

__global__ void __launch_bounds__(32) bz2_parse_kernel(Batch b) {
  __shared__ Bz2State st;
  if (threadIdx.x) return;
  Bz2View v(b, blockIdx.x);
  const uint64_t src_size = v.d->src_size;
  const Bz2Caps cap = bz2Caps(v.d->dst_size);
  uint32_t nb = 0, comb = 0;
  const int32_t r = bz2_parse(b.base + v.d->src, src_size, st, v.tt, cap, v.blk, &nb, &comb);
  v.d->nb = r ? 0 : nb;
  v.d->comb = comb;
  if (r) v.d->reason = r;
}

// tile t of the chunk: its block and its position range in that block; false if there is no such tile
__device__ bool tileOf(const Bz2View& v, uint32_t t, uint32_t* blk, uint32_t* lo, uint32_t* hi) {
  const uint32_t k = v.find(t, false);
  if (k >= v.d->nb) return false;
  const Bz2Block& B = v.blk[k];
  *blk = k;
  *lo = (t - B.tile0) * kTile;
  *hi = min(B.nblock, *lo + kTile);
  return true;
}

__global__ void __launch_bounds__(32) bz2_hist_kernel(Batch b) {
  __shared__ uint32_t h[256 * 32];
  Bz2View v(b, blockIdx.y);
  const uint32_t t = blockIdx.x * 32 + threadIdx.x;
  uint32_t k, lo, hi;
  if (v.d->reason || !tileOf(v, t, &k, &lo, &hi)) return;
  for (int s = 0; s < 256; ++s) h[s * 32 + threadIdx.x] = 0;
  bz2_tile_count(v.tt + v.blk[k].tt_off, lo, hi, h + threadIdx.x, 32);
  uint32_t* out = v.hist + (size_t)t * 256;
  for (int s = 0; s < 256; ++s) out[s] = h[s * 32 + threadIdx.x];
}

__global__ void __launch_bounds__(256) bz2_scan_kernel(Batch b) {
  __shared__ uint32_t tot[256];
  Bz2View v(b, blockIdx.y);
  if (v.d->reason || blockIdx.x >= v.d->nb) return;
  const Bz2Block& B = v.blk[blockIdx.x];
  uint32_t* h = v.hist + (size_t)B.tile0 * 256;
  tot[threadIdx.x] = bz2_scan_symbol(h, B.ntiles, threadIdx.x);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t acc = 0;
    for (int s = 0; s < 256; ++s) { const uint32_t c = tot[s]; tot[s] = acc; acc += c; }
  }
  __syncthreads();
  bz2_scan_add(h, B.ntiles, threadIdx.x, tot[threadIdx.x]);
}

__global__ void __launch_bounds__(32) bz2_scatter_kernel(Batch b) {
  __shared__ uint32_t pos[256 * 32];
  Bz2View v(b, blockIdx.y);
  const uint32_t t = blockIdx.x * 32 + threadIdx.x;
  uint32_t k, lo, hi;
  if (v.d->reason || !tileOf(v, t, &k, &lo, &hi)) return;
  const uint32_t* in = v.hist + (size_t)t * 256;
  for (int s = 0; s < 256; ++s) pos[s * 32 + threadIdx.x] = in[s];
  bz2_tile_scatter(v.tt + v.blk[k].tt_off, lo, hi, pos + threadIdx.x, 32);
}

__global__ void __launch_bounds__(128) bz2_walk_len_kernel(Batch b) {
  Bz2View v(b, blockIdx.y);
  const uint32_t g = blockIdx.x * 128 + threadIdx.x;
  if (v.d->reason) return;
  const uint32_t k = v.find(g, true);
  if (k >= v.d->nb) return;
  const Bz2Block& B = v.blk[k];
  if (!bz2_walk_len(v.tt + B.tt_off, B, g - B.samp0, v.slen + g, v.ssucc + g)) fail(&v.d->reason, BZ_BWT);
}

__global__ void __launch_bounds__(32) bz2_order_kernel(Batch b) {
  Bz2View v(b, blockIdx.y);
  const uint32_t k = blockIdx.x * 32 + threadIdx.x;
  if (v.d->reason || k >= v.d->nb) return;
  Bz2Block& B = v.blk[k];
  if (!bz2_order(v.tt + B.tt_off, B, v.slen + B.samp0, v.ssucc + B.samp0, v.soff + B.samp0)) fail(&v.d->reason, BZ_BWT);
}

__global__ void __launch_bounds__(128) bz2_walk_write_kernel(Batch b) {
  Bz2View v(b, blockIdx.y);
  const uint32_t g = blockIdx.x * 128 + threadIdx.x;
  if (v.d->reason) return;
  const uint32_t k = v.find(g, true);
  if (k >= v.d->nb || v.soff[g] == kAbsentSample) return;
  const Bz2Block& B = v.blk[k];
  bz2_walk_write(v.tt + B.tt_off, B, g - B.samp0, v.slen[g], v.soff[g], v.pre + B.tt_off);
}

template <bool kWrite>
__device__ void unrle(const Batch& b) {
  __shared__ uint32_t tab[256];
  for (int i = threadIdx.x; i < 256; i += 32) tab[i] = crcEntry(i);
  __syncthreads();
  Bz2View v(b, blockIdx.y);
  const uint32_t k = blockIdx.x * 32 + threadIdx.x;
  if (v.d->reason || k >= v.d->nb) return;
  Bz2Block& B = v.blk[k];
  if (kWrite) {
    uint32_t crc;
    bz2_unrle(v.pre + B.tt_off, B.nblock, b.base + v.d->dst + B.out_off, B.out_len, tab, &crc);
  } else {
    const int64_t n = bz2_unrle(v.pre + B.tt_off, B.nblock, nullptr, v.d->dst_size, tab, &B.crc_calc);
    if (n < 0) fail(&v.d->reason, BZ_SIZE);
    else B.out_len = (uint32_t)n;
  }
}
__global__ void __launch_bounds__(32) bz2_unrle_count_kernel(Batch b) { unrle<false>(b); }
__global__ void __launch_bounds__(32) bz2_unrle_write_kernel(Batch b) { unrle<true>(b); }

__global__ void __launch_bounds__(32) bz2_finish_kernel(Batch b, uint32_t nbz) {
  const uint32_t k = blockIdx.x * 32 + threadIdx.x;
  if (k >= nbz) return;
  Bz2View v(b, k);
  if (v.d->reason) return;
  const int32_t r = bz2_finish(v.blk, v.d->nb, v.d->comb, v.d->dst_size);
  if (r) v.d->reason = r;
}

__global__ void __launch_bounds__(32) lz4_frame_kernel(Batch b) {
  Desc* d = &b.desc[b.lz[blockIdx.x]];
  const int32_t r = lz4_frame(b.base + d->src, d->src_size, b.base + d->dst, d->dst_size, threadIdx.x, 32);
  if (threadIdx.x == 0 && r) d->reason = r;
}

size_t workBytes(const esvo_chunk& c) { return c.codec == ESVO_CODEC_BZ2 ? Layout(bz2Caps(c.dst_size)).bytes : 0; }
size_t chunkBytes(const esvo_chunk& c) { return alignUp(c.src_size) + alignUp(c.dst_size) + workBytes(c); }
size_t headBytes(size_t n) { return alignUp(n * (sizeof(Desc) + 8)); }

int codeOf(int32_t reason) { return reason >= R_FIRST_UNSUPPORTED ? ESVO_ERR_UNSUPPORTED : ESVO_ERR_INVALID_ARG; }

}  // namespace esvo_inflate

using namespace esvo_inflate;

struct esvo_inflater {
  int device = 0;
  cudaStream_t stream = nullptr;
  uint8_t* scratch = nullptr;
  size_t scratch_bytes = 0;
  uint8_t* pinned = nullptr;
  size_t pinned_bytes = 0;
  std::string err;
};

extern "C" {

ESVO_API int esvo_inflater_create(int device, size_t scratch_bytes, esvo_inflater** out) {
  if (!out) return ESVO_ERR_INVALID_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    cudaGetLastError();
    return ESVO_ERR_NO_DEVICE;
  }
  if (scratch_bytes < kAlign) return ESVO_ERR_INVALID_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return ESVO_ERR_NO_DEVICE;
  esvo_inflater* inf = new esvo_inflater;
  inf->device = device;
  inf->scratch_bytes = scratch_bytes;
  if (cudaStreamCreateWithFlags(&inf->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMalloc(&inf->scratch, scratch_bytes) != cudaSuccess) {
    cudaGetLastError();
    esvo_inflater_destroy(inf);
    return ESVO_ERR_CUDA;
  }
  *out = inf;
  return ESVO_OK;
}

ESVO_API void esvo_inflater_destroy(esvo_inflater* inf) {
  if (!inf) return;
  cudaSetDevice(inf->device);
  if (inf->stream) cudaStreamSynchronize(inf->stream);
  cudaFree(inf->scratch);
  cudaFreeHost(inf->pinned);
  if (inf->stream) cudaStreamDestroy(inf->stream);
  delete inf;
}

ESVO_API const char* esvo_inflater_last_error(const esvo_inflater* inf) { return inf ? inf->err.c_str() : "no inflater"; }

ESVO_API int esvo_inflate_chunks(esvo_inflater* inf, esvo_chunk* chunks, int n) {
  if (!inf) return ESVO_ERR_INVALID_ARG;
  inf->err.clear();
  if (n < 0 || (n > 0 && !chunks)) { inf->err = "esvo_inflate_chunks: invalid chunk list"; return ESVO_ERR_INVALID_ARG; }
  if (cudaSetDevice(inf->device) != cudaSuccess) { inf->err = "esvo_inflate_chunks: cannot select the device"; return ESVO_ERR_CUDA; }
  std::vector<std::string> why(n);
  auto refuse = [&](int i, int code, const std::string& text) { chunks[i].status = code; why[i] = text; };
  auto result = [&]() {   // the first failing chunk's code and reason
    for (int i = 0; i < n; ++i)
      if (chunks[i].status != ESVO_OK) { inf->err = "chunk " + std::to_string(i) + ": " + why[i]; return (int)chunks[i].status; }
    return (int)ESVO_OK;
  };
  // the chunks to run, in order; refused up front: bad arguments, unknown codecs, chunks larger than the scratch
  std::vector<int> todo;
  for (int i = 0; i < n; ++i) {
    esvo_chunk& c = chunks[i];
    c.status = ESVO_OK;
    if ((!c.src && c.src_size) || (!c.dst && c.dst_size) || c.dst_size > 0xC0000000ull) {
      refuse(i, ESVO_ERR_INVALID_ARG, "null buffer or a size past 3 GiB");
    } else if (c.codec != ESVO_CODEC_BZ2 && c.codec != ESVO_CODEC_LZ4) {
      refuse(i, ESVO_ERR_UNSUPPORTED, "unknown codec " + std::to_string(c.codec));
    } else if (headBytes(1) + chunkBytes(c) > inf->scratch_bytes) {
      refuse(i, ESVO_ERR_CAPACITY, "needs " + std::to_string(headBytes(1) + chunkBytes(c)) + " bytes of scratch, the inflater has " +
                                       std::to_string(inf->scratch_bytes));
    } else {
      todo.push_back(i);
    }
  }
  auto cuda_fail = [&](cudaError_t e) {
    cudaGetLastError();
    inf->err = std::string("esvo_inflate_chunks: ") + cudaGetErrorString(e);
    const std::string msg = inf->err;
    for (int i : todo) if (chunks[i].status == ESVO_OK) chunks[i].status = ESVO_ERR_CUDA;
    inf->err = msg;
    return ESVO_ERR_CUDA;
  };
  size_t a = 0;
  while (a < todo.size()) {
    // the batch [a, e): as many chunks as fit
    size_t e = a, body = 0;
    while (e < todo.size() && e - a < 65535 &&
           headBytes(e - a + 1) + body + chunkBytes(chunks[todo[e]]) <= inf->scratch_bytes) body += chunkBytes(chunks[todo[e++]]);
    const size_t m = e - a, head = headBytes(m);
    std::vector<Desc> desc(m);
    std::vector<uint32_t> bz, lz;
    size_t src_end = head, dst_end, work_end;
    for (size_t k = 0; k < m; ++k) { desc[k].src = src_end; src_end += alignUp(chunks[todo[a + k]].src_size); }
    dst_end = src_end;
    for (size_t k = 0; k < m; ++k) { desc[k].dst = dst_end; dst_end += alignUp(chunks[todo[a + k]].dst_size); }
    work_end = dst_end;
    uint32_t max_tiles = 0, max_samp = 0, max_nb = 0;
    for (size_t k = 0; k < m; ++k) {
      const esvo_chunk& c = chunks[todo[a + k]];
      Desc& d = desc[k];
      d.src_size = c.src_size; d.dst_size = c.dst_size; d.codec = c.codec; d.reason = 0; d.nb = 0; d.comb = 0;
      d.work = work_end;
      work_end += workBytes(c);
      if (c.codec == ESVO_CODEC_BZ2) {
        bz.push_back((uint32_t)k);
        const Bz2Caps cap = bz2Caps(c.dst_size);
        max_tiles = std::max(max_tiles, cap.tiles); max_samp = std::max(max_samp, cap.samp); max_nb = std::max(max_nb, cap.nb);
      } else {
        lz.push_back((uint32_t)k);
      }
    }
    const size_t down = head + (dst_end - src_end);
    if (std::max(src_end, down) > inf->pinned_bytes) {
      cudaFreeHost(inf->pinned);
      inf->pinned = nullptr; inf->pinned_bytes = 0;
      const size_t want = std::max(src_end, down);
      if (cudaError_t r = cudaHostAlloc(&inf->pinned, want, cudaHostAllocDefault)) return cuda_fail(r);
      inf->pinned_bytes = want;
    }
    uint8_t* pin = inf->pinned;
    std::memcpy(pin, desc.data(), m * sizeof(Desc));
    std::memcpy(pin + m * sizeof(Desc), bz.data(), bz.size() * 4);
    std::memcpy(pin + m * sizeof(Desc) + bz.size() * 4, lz.data(), lz.size() * 4);
    for (size_t k = 0; k < m; ++k)
      if (desc[k].src_size) std::memcpy(pin + desc[k].src, chunks[todo[a + k]].src, desc[k].src_size);
    cudaStream_t s = inf->stream;
    if (cudaError_t r = cudaMemcpyAsync(inf->scratch, pin, src_end, cudaMemcpyHostToDevice, s)) return cuda_fail(r);
    Batch bt{inf->scratch, (Desc*)inf->scratch, (const uint32_t*)(inf->scratch + m * sizeof(Desc)),
             (const uint32_t*)(inf->scratch + m * sizeof(Desc) + bz.size() * 4)};
    const uint32_t nbz = (uint32_t)bz.size();
    if (nbz) {
      const dim3 tiles((max_tiles + 31) / 32, nbz), samp((max_samp + 127) / 128, nbz), blocks((max_nb + 31) / 32, nbz);
      bz2_parse_kernel<<<nbz, 32, 0, s>>>(bt);
      bz2_hist_kernel<<<tiles, 32, 0, s>>>(bt);
      bz2_scan_kernel<<<dim3(max_nb, nbz), 256, 0, s>>>(bt);
      bz2_scatter_kernel<<<tiles, 32, 0, s>>>(bt);
      bz2_walk_len_kernel<<<samp, 128, 0, s>>>(bt);
      bz2_order_kernel<<<blocks, 32, 0, s>>>(bt);
      bz2_walk_write_kernel<<<samp, 128, 0, s>>>(bt);
      bz2_unrle_count_kernel<<<blocks, 32, 0, s>>>(bt);
      bz2_finish_kernel<<<(nbz + 31) / 32, 32, 0, s>>>(bt, nbz);
      bz2_unrle_write_kernel<<<blocks, 32, 0, s>>>(bt);
    }
    if (!lz.empty()) lz4_frame_kernel<<<(unsigned)lz.size(), 32, 0, s>>>(bt);
    if (cudaError_t r = cudaGetLastError()) return cuda_fail(r);
    // descriptors first (into the head of the staging), then the outputs behind them
    if (cudaError_t r = cudaMemcpyAsync(pin, inf->scratch, m * sizeof(Desc), cudaMemcpyDeviceToHost, s)) return cuda_fail(r);
    if (dst_end > src_end)
      if (cudaError_t r = cudaMemcpyAsync(pin + head, inf->scratch + src_end, dst_end - src_end, cudaMemcpyDeviceToHost, s))
        return cuda_fail(r);
    if (cudaError_t r = cudaStreamSynchronize(s)) return cuda_fail(r);
    std::memcpy(desc.data(), pin, m * sizeof(Desc));
    for (size_t k = 0; k < m; ++k) {
      const int i = todo[a + k];
      if (desc[k].reason) { refuse(i, codeOf(desc[k].reason), reasonText(desc[k].reason)); continue; }
      if (desc[k].dst_size) std::memcpy(chunks[i].dst, pin + head + (desc[k].dst - src_end), desc[k].dst_size);
    }
    a = e;
  }
  return result();
}

}  // extern "C"
