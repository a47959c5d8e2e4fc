// esvo_b200 product code -- the bz2 and LZ4 chunk decoders of a compressed ROS bag (include/esvo_b200_inflate.h).
//
// Every stage is a per-work-item function (INF_HD = host + device): inflate.cu launches them as CUDA threads / warps;
// tests/inflate_host_check.cpp runs the very same functions in plain loops, so the decoders are verified byte for byte
// against Python's bz2 (libbz2) and an LZ4 frame writer built from the format description, sanitizers included, where no
// GPU is available.
//
// bz2 (one bzip2 stream per chunk), in the stages inflate.cu runs:
//   (a) bz2_parse            one thread per chunk: stream and block headers, Huffman / MTF / RUNA-RUNB symbol decode of
//                            every block into the L column of its BWT (tt[i] = byte, the libbz2 layout);
//   (b) bz2_tile_count, bz2_scan_symbol, bz2_tile_scatter
//                            the inverse-BWT vector by a stable counting sort: per-tile histograms, a scan over the tiles
//                            of a block, then each tile scatters its positions: tt[cftab[L[i]] + rank] |= i << 8;
//   (c) bz2_walk_len, bz2_order, bz2_walk_write
//                            the inverse-BWT walk from one sample per kStride positions (plus the start position): each
//                            walk stops at the next sample, the segments are chained by their successor samples, and a
//                            second walk writes every segment at its offset -- 2 * nblock steps in nblock / kStride
//                            independent chains instead of one chain of nblock dependent loads (a periodic block's
//                            output repeats the cycle through the start position);
//   (d) bz2_unrle            one thread per block: undo the initial run-length coding, count (and CRC) or write;
//       bz2_finish           one thread per chunk: block CRCs, combined CRC, output offsets and the declared size.
// LZ4 (one frame per chunk, format v1.6): lz4_frame decodes a whole frame; run by `nl` lanes, every lane parses the same
// tokens and the lanes share each literal / match copy (a match copies from out[pos - off + i % off], already written).
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define INF_HD __host__ __device__ __forceinline__
#else
#define INF_HD inline
#endif
#ifdef __CUDA_ARCH__
#define INF_SYNC() __syncwarp()
#else
#define INF_SYNC() ((void)0)
#endif

namespace esvo_inflate {

// ---------------------------------------------------------------- refusals
enum Reason : int32_t {
  R_OK = 0,
  // invalid streams (ESVO_ERR_INVALID_ARG)
  BZ_MAGIC, BZ_BLOCK_MAGIC, BZ_TRUNCATED, BZ_NO_SYMBOLS, BZ_GROUPS, BZ_SELECTORS, BZ_CODE_LENGTHS, BZ_HUFFMAN,
  BZ_BLOCK_SIZE, BZ_RUN, BZ_ORIG_PTR, BZ_BWT, BZ_BLOCK_CRC, BZ_STREAM_CRC, BZ_TRAILING, BZ_SIZE,
  LZ4_MAGIC, LZ4_DESCRIPTOR, LZ4_HEADER_CHECKSUM, LZ4_TRUNCATED, LZ4_BLOCK_SIZE, LZ4_OFFSET, LZ4_OVERFLOW,
  LZ4_BLOCK_CHECKSUM, LZ4_CONTENT_CHECKSUM, LZ4_SIZE, LZ4_TRAILING,
  // unsupported streams (ESVO_ERR_UNSUPPORTED)
  R_FIRST_UNSUPPORTED,
  BZ_RANDOMISED = R_FIRST_UNSUPPORTED, BZ_TOO_MANY_BLOCKS, LZ4_LEGACY, LZ4_SKIPPABLE, LZ4_DICT_ID, R_CODEC,
  R_COUNT
};

inline const char* reasonText(int32_t r) {
  static const char* const t[R_COUNT] = {
      "ok",
      "bz2: not a bzip2 stream (no BZh1..BZh9 header)",
      "bz2: bad block or end-of-stream magic",
      "bz2: truncated stream",
      "bz2: block uses no symbols",
      "bz2: number of Huffman groups not in 2..6",
      "bz2: bad selectors",
      "bz2: code length not in 1..20",
      "bz2: invalid Huffman code",
      "bz2: block larger than the stream's block size",
      "bz2: run overflows the block",
      "bz2: origPtr outside the block",
      "bz2: inverse BWT does not close into a cycle",
      "bz2: block CRC mismatch",
      "bz2: combined stream CRC mismatch",
      "bz2: data after the end of the stream",
      "bz2: decompressed size differs from the chunk's size",
      "lz4: not an LZ4 frame",
      "lz4: invalid frame descriptor",
      "lz4: frame header checksum mismatch",
      "lz4: truncated frame",
      "lz4: block larger than the frame's block size",
      "lz4: match offset before the start of the output",
      "lz4: output larger than the chunk's size",
      "lz4: block checksum mismatch",
      "lz4: content checksum mismatch",
      "lz4: decompressed size differs from the chunk's size",
      "lz4: data after the end of the frame",
      "bz2: randomised block (bzip2 < 0.9.5) is not supported",
      "bz2: more blocks than a bzip2 compressor writes for this size",
      "lz4: legacy frames are not supported",
      "lz4: skippable frames are not supported",
      "lz4: frames with a dictionary ID are not supported",
      "unknown codec",
  };
  return r >= 0 && r < R_COUNT ? t[r] : "?";
}

INF_HD void fail(int32_t* reason, int32_t r) {   // keeps the first refusal of a chunk
#ifdef __CUDA_ARCH__
  atomicCAS(reason, 0, r);
#else
  if (*reason == 0) *reason = r;
#endif
}

// ---------------------------------------------------------------- bz2 layout
constexpr uint32_t kTile = 2048;      // positions per counting-sort tile
constexpr uint32_t kStride = 1024;    // positions per inverse-BWT sample
constexpr uint32_t kMaxSelectors = 18002;
constexpr uint32_t kAbsentSample = 0xffffffffu;

struct Bz2Block {
  uint32_t tt_off;     // first position of the block in the chunk's tt / pre arrays
  uint32_t nblock;     // positions (bytes before the initial-RLE undo)
  uint32_t orig_ptr;
  uint32_t crc;        // stored block CRC
  uint32_t tile0, ntiles;   // the block's tiles in the chunk's histogram array
  uint32_t samp0, nsamp;    // the block's samples in the chunk's sample arrays (nsamp = ceil(nblock / kStride) + 1)
  uint32_t cycle;      // length of p0's inverse-BWT cycle (stage c)
  uint32_t crc_calc;   // CRC of the decoded bytes (stage d)
  uint32_t out_len;    // decoded bytes (stage d)
  uint64_t out_off;    // offset in the chunk's output (bz2_finish)
};

// Worst-case work sizes of a chunk, from its sizes alone.  A block's nblock is at most 5/4 of its output plus one (the
// initial RLE turns 4 equal bytes into 4 bytes and a count); a bzip2 compressor fills every block but the last, so a
// stream of dst bytes has at most dst / 32768 + 4 blocks (a stream with more is refused as unsupported).
struct Bz2Caps { uint32_t nb, tt, tiles, samp; };
INF_HD Bz2Caps bz2Caps(uint64_t dst_size) {
  Bz2Caps c;
  c.nb = (uint32_t)(dst_size / 32768 + 4);
  c.tt = (uint32_t)(dst_size + dst_size / 4 + c.nb);
  c.tiles = c.tt / kTile + c.nb;
  c.samp = c.tt / kStride + 2 * c.nb;
  return c;
}

INF_HD uint32_t crcEntry(uint32_t i) {   // CRC-32, polynomial 0x04C11DB7, MSB first
  uint32_t c = i << 24;
  for (int k = 0; k < 8; ++k) c = (c & 0x80000000u) ? (c << 1) ^ 0x04C11DB7u : c << 1;
  return c;
}
INF_HD uint32_t crcByte(const uint32_t* tab, uint32_t crc, uint32_t b) { return (crc << 8) ^ tab[(crc >> 24) ^ b]; }

// ---------------------------------------------------------------- bit reader (MSB first)
struct Bits {
  const uint8_t* p;
  uint64_t n, pos;     // bytes, next byte
  uint64_t buf;
  int cnt;
  bool over;           // read past the end (zeros were supplied)
  INF_HD uint32_t get(int k) {   // k <= 24
    while (cnt < k) {
      buf = (buf << 8) | (pos < n ? p[pos] : 0);
      if (pos >= n) over = true;
      ++pos; cnt += 8;
    }
    cnt -= k;
    return (uint32_t)(buf >> cnt) & ((1u << k) - 1u);
  }
  INF_HD uint32_t bit() { return get(1); }
  INF_HD uint32_t get32() { const uint32_t h = get(16); return (h << 16) | get(16); }
};

// Per-chunk state of the symbol decode (shared memory on the device: about 20 KB)
struct Bz2State {
  uint8_t sel[kMaxSelectors];
  uint8_t len[6][258];
  uint16_t perm[6][258];
  int32_t first[6][22];   // canonical code of the first symbol of each length
  int32_t count[6][22];
  int32_t index[6][22];   // position of that symbol in perm
  int32_t minl[6], maxl[6];
  uint8_t unseq[256];
  uint8_t mtf[256];
};

// Huffman code of group g from len[g][0..a): canonical, ordered by length then symbol (as bzip2 assigns them).
// Oversubscribed codes are refused.
INF_HD bool bz2Tables(Bz2State& s, int g, int a) {
  int mn = 32, mx = 0;
  for (int i = 0; i < 22; ++i) s.count[g][i] = 0;
  for (int i = 0; i < a; ++i) {
    const int l = s.len[g][i];
    mn = l < mn ? l : mn; mx = l > mx ? l : mx;
    ++s.count[g][l];
  }
  int code = 0, idx = 0;
  for (int l = 1; l <= 20; ++l) {
    s.first[g][l] = code;
    s.index[g][l] = idx;
    code += s.count[g][l];
    if (code > (1 << l)) return false;
    idx += s.count[g][l];
    code <<= 1;
  }
  int k = 0;
  for (int l = mn; l <= mx; ++l)
    for (int i = 0; i < a; ++i)
      if (s.len[g][i] == l) s.perm[g][k++] = (uint16_t)i;
  s.minl[g] = mn; s.maxl[g] = mx;
  return true;
}

INF_HD int bz2Symbol(Bz2State& s, Bits& b, int g) {   // -1: no code matches
  int l = s.minl[g];
  uint32_t v = b.get(l);
  for (;;) {
    const uint32_t d = v - (uint32_t)s.first[g][l];
    if (d < (uint32_t)s.count[g][l]) return s.perm[g][s.index[g][l] + d];
    if (++l > s.maxl[g]) return -1;
    v = (v << 1) | b.bit();
  }
}

// (a) Decodes the headers and symbols of every block of the stream src[0, n): block b's L column goes to
// tt[blk[b].tt_off ...] (one byte per u32 word, the upper 24 bits zero), its tiles and samples are numbered.  Returns
// R_OK or the refusal.  *nb_out = blocks, *comb_out = the stored combined CRC.
INF_HD int32_t bz2_parse(const uint8_t* src, uint64_t n, Bz2State& s, uint32_t* tt, const Bz2Caps& cap, Bz2Block* blk,
                         uint32_t* nb_out, uint32_t* comb_out) {
  Bits b{src, n, 0, 0, 0, false};
  *nb_out = 0;
  if (n < 4 || src[0] != 'B' || src[1] != 'Z' || src[2] != 'h' || src[3] < '1' || src[3] > '9') return BZ_MAGIC;
  b.pos = 4;
  const uint32_t max_block = (uint32_t)(src[3] - '0') * 100000u;
  uint32_t nb = 0, tt_used = 0, tiles = 0, samp = 0;
  for (;;) {
    const uint32_t m1 = b.get(24), m2 = b.get(24);
    if (b.over) return BZ_TRUNCATED;
    if (m1 == 0x177245 && m2 == 0x385090) {             // end of stream
      *comb_out = b.get32();
      if (b.over) return BZ_TRUNCATED;
      if (b.cnt > 0 && (b.buf & ((1ull << b.cnt) - 1)) != 0) return BZ_TRAILING;   // padding of the last byte
      if (b.pos != n) return BZ_TRAILING;
      *nb_out = nb;
      return R_OK;
    }
    if (m1 != 0x314159 || m2 != 0x265359) return BZ_BLOCK_MAGIC;
    if (nb == cap.nb) return BZ_TOO_MANY_BLOCKS;
    Bz2Block& B = blk[nb];
    B.crc = b.get32();
    if (b.bit()) return b.over ? BZ_TRUNCATED : BZ_RANDOMISED;
    B.orig_ptr = b.get(24);
    // symbol map
    const uint32_t used16 = b.get(16);
    int n_in_use = 0;
    for (int i = 0; i < 16; ++i)
      if (used16 & (0x8000u >> i)) {
        const uint32_t u = b.get(16);
        for (int j = 0; j < 16; ++j)
          if (u & (0x8000u >> j)) s.unseq[n_in_use++] = (uint8_t)(i * 16 + j);
      }
    if (b.over) return BZ_TRUNCATED;
    if (n_in_use == 0) return BZ_NO_SYMBOLS;
    const int alpha = n_in_use + 2;
    const int n_groups = (int)b.get(3);
    if (n_groups < 2 || n_groups > 6) return BZ_GROUPS;
    uint32_t n_sel = b.get(15);
    if (n_sel < 1) return BZ_SELECTORS;
    // selectors: MTF-coded unary; beyond kMaxSelectors read and ignored
    uint8_t pos[6];
    for (int i = 0; i < 6; ++i) pos[i] = (uint8_t)i;
    for (uint32_t i = 0; i < n_sel; ++i) {
      int j = 0;
      while (b.bit()) {
        if (++j >= n_groups) return BZ_SELECTORS;
        if (b.over) return BZ_TRUNCATED;
      }
      if (i < kMaxSelectors) {
        const uint8_t v = pos[j];
        for (; j > 0; --j) pos[j] = pos[j - 1];
        pos[0] = v;
        s.sel[i] = v;
      }
    }
    if (b.over) return BZ_TRUNCATED;
    if (n_sel > kMaxSelectors) n_sel = kMaxSelectors;
    // delta-coded code lengths
    for (int g = 0; g < n_groups; ++g) {
      int c = (int)b.get(5);
      for (int i = 0; i < alpha; ++i) {
        for (;;) {
          if (c < 1 || c > 20) return BZ_CODE_LENGTHS;
          if (!b.bit()) break;
          c += b.bit() ? -1 : 1;
          if (b.over) return BZ_TRUNCATED;
        }
        s.len[g][i] = (uint8_t)c;
      }
      if (!bz2Tables(s, g, alpha)) return BZ_HUFFMAN;
    }
    if (b.over) return BZ_TRUNCATED;
    // symbols: RUNA / RUNB runs of the front symbol, MTF indices, end of block
    for (int i = 0; i < n_in_use; ++i) s.mtf[i] = (uint8_t)i;
    const uint32_t limit = max_block < cap.tt - tt_used ? max_block : cap.tt - tt_used;
    uint32_t* out = tt + tt_used;
    uint32_t nblock = 0, run = 0, run_w = 1, gsel = 0, left = 0;
    int g = 0;
    const int eob = n_in_use + 1;
    for (;;) {
      if (left == 0) {
        if (gsel >= n_sel) return BZ_SELECTORS;
        g = s.sel[gsel++]; left = 50;
        if (g >= n_groups) return BZ_SELECTORS;
      }
      --left;
      const int sym = bz2Symbol(s, b, g);
      if (b.over) return BZ_TRUNCATED;
      if (sym < 0) return BZ_HUFFMAN;
      if (sym <= 1) {                                     // RUNA = 1 * w, RUNB = 2 * w
        if (run_w >= (1u << 21)) return BZ_RUN;
        run += (uint32_t)(sym + 1) * run_w;
        run_w <<= 1;
        continue;
      }
      if (run) {
        if (run > limit - nblock) return BZ_RUN;
        const uint32_t v = s.unseq[s.mtf[0]];
        for (uint32_t k = 0; k < run; ++k) out[nblock + k] = v;
        nblock += run; run = 0;
      }
      run_w = 1;
      if (sym == eob) break;
      if (nblock >= limit) return BZ_BLOCK_SIZE;
      int j = sym - 1;                                    // MTF index 1 .. n_in_use - 1
      const uint8_t v = s.mtf[j];
      for (; j > 0; --j) s.mtf[j] = s.mtf[j - 1];
      s.mtf[0] = v;
      out[nblock++] = s.unseq[v];
    }
    if (B.orig_ptr >= nblock) return BZ_ORIG_PTR;
    B.tt_off = tt_used; B.nblock = nblock;
    B.tile0 = tiles; B.ntiles = (nblock + kTile - 1) / kTile;
    B.samp0 = samp; B.nsamp = (nblock + kStride - 1) / kStride + 1;
    tt_used += nblock; tiles += B.ntiles; samp += B.nsamp;
    ++nb;
  }
}

// (b) counting sort of one block's L column into its inverse-BWT vector.  hist holds 256 counters per tile, at stride hs.
INF_HD void bz2_tile_count(const uint32_t* tt, uint32_t b, uint32_t e, uint32_t* h, int hs) {
  for (uint32_t i = b; i < e; ++i) ++h[(tt[i] & 255u) * hs];
}
// Tile counts of symbol `sym` (hist[t * 256 + sym], t < ntiles) -> exclusive prefix over the tiles; returns the total.
INF_HD uint32_t bz2_scan_symbol(uint32_t* hist, uint32_t ntiles, int sym) {
  uint32_t acc = 0;
  for (uint32_t t = 0; t < ntiles; ++t) { const uint32_t c = hist[t * 256 + sym]; hist[t * 256 + sym] = acc; acc += c; }
  return acc;
}
INF_HD void bz2_scan_add(uint32_t* hist, uint32_t ntiles, int sym, uint32_t base) {
  for (uint32_t t = 0; t < ntiles; ++t) hist[t * 256 + sym] += base;
}
// tt[pos[L[i]]++] |= i << 8 for i in [b, e): pos at stride ps, the tile's first position of each symbol
INF_HD void bz2_tile_scatter(uint32_t* tt, uint32_t b, uint32_t e, uint32_t* pos, int ps) {
  for (uint32_t i = b; i < e; ++i) {
    const uint32_t s = tt[i] & 255u;
    tt[pos[s * ps]++] |= i << 8;
  }
}

// (c) the inverse-BWT walk.  The output starts at p0 = tt[orig_ptr] >> 8 and steps q -> tt[q] >> 8 emitting tt[q] & 255.
// Samples: k * kStride for k < ns = ceil(nblock / kStride), and p0 as sample ns (unused when p0 is a multiple of kStride).
INF_HD uint32_t bz2_p0(const uint32_t* tt, const Bz2Block& B) { return tt[B.orig_ptr] >> 8; }
INF_HD uint32_t bz2_sample_id(uint32_t q, uint32_t p0, uint32_t ns) {
  return q % kStride == 0 ? q / kStride : (q == p0 ? ns : kAbsentSample);
}
// Walks sample j until the next sample: its length and successor (kAbsentSample for the unused sample); false if the walk
// leaves the block or does not reach a sample within nblock steps.
INF_HD bool bz2_walk_len(const uint32_t* tt, const Bz2Block& B, uint32_t j, uint32_t* len, uint32_t* succ) {
  const uint32_t p0 = bz2_p0(tt, B), ns = B.nsamp - 1;
  *len = 0; *succ = kAbsentSample;
  uint32_t q;
  if (j == ns) { if (p0 % kStride == 0) return true; q = p0; }
  else q = j * kStride;
  for (uint32_t l = 1; l <= B.nblock; ++l) {
    q = tt[q] >> 8;
    if (q >= B.nblock) return false;
    const uint32_t id = bz2_sample_id(q, p0, ns);
    if (id != kAbsentSample) { *len = l; *succ = id; return true; }
  }
  return false;
}
// Chains the segments of p0's cycle from p0's sample: soff = each sample's offset in the cycle, B.cycle = its length.  A
// periodic block has several cycles; its output is p0's cycle repeated (nblock steps from p0), so samples off that cycle
// stay absent.  False if the successor links do not close into a cycle.
INF_HD bool bz2_order(const uint32_t* tt, Bz2Block& B, const uint32_t* slen, const uint32_t* ssucc, uint32_t* soff) {
  const uint32_t p0 = bz2_p0(tt, B), ns = B.nsamp - 1;
  for (uint32_t j = 0; j < B.nsamp; ++j) soff[j] = kAbsentSample;
  const uint32_t start = bz2_sample_id(p0, p0, ns);
  uint32_t cur = start, off = 0;
  for (uint32_t k = 0; k < B.nsamp; ++k) {
    if (cur >= B.nsamp || soff[cur] != kAbsentSample || slen[cur] == 0 || slen[cur] > B.nblock - off) return false;
    soff[cur] = off; off += slen[cur];
    cur = ssucc[cur];
    if (cur == start) { B.cycle = off; return true; }
  }
  return false;
}
// Writes sample j's segment at its offset in every repetition of the cycle within the block.
INF_HD void bz2_walk_write(const uint32_t* tt, const Bz2Block& B, uint32_t j, uint32_t len, uint32_t off, uint8_t* pre) {
  const uint32_t ns = B.nsamp - 1;
  uint32_t q = j == ns ? bz2_p0(tt, B) : j * kStride;
  for (uint32_t l = 0; l < len; ++l) {
    const uint32_t e = tt[q];
    for (uint32_t p = off + l; p < B.nblock; p += B.cycle) pre[p] = (uint8_t)e;
    q = e >> 8;
  }
}

// (d) undoes the initial RLE (4 equal bytes, then a count of further copies; never across a block) of pre[0, n):
// out == nullptr counts; otherwise writes.  Returns the decoded length, or -1 once it would pass cap.  *crc: the block CRC.
INF_HD int64_t bz2_unrle(const uint8_t* pre, uint32_t n, uint8_t* out, uint64_t cap, const uint32_t* tab, uint32_t* crc) {
  uint64_t o = 0;
  uint32_t c = 0xffffffffu;
  int last = -1, run = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t v = pre[i];
    if (run == 4) {
      if (v > cap - o) return -1;
      for (uint32_t k = 0; k < v; ++k) c = crcByte(tab, c, (uint32_t)last);
      if (out) for (uint32_t k = 0; k < v; ++k) out[o + k] = (uint8_t)last;
      o += v; run = 0; last = -1;
      continue;
    }
    if (o >= cap) return -1;
    c = crcByte(tab, c, v);
    if (out) out[o] = (uint8_t)v;
    ++o;
    if ((int)v == last) ++run; else { last = (int)v; run = 1; }
  }
  *crc = ~c;
  return (int64_t)o;
}

// Block CRCs, combined CRC and output offsets of a chunk whose blocks have been counted.
INF_HD int32_t bz2_finish(Bz2Block* blk, uint32_t nb, uint32_t stored_comb, uint64_t dst_size) {
  uint32_t comb = 0;
  uint64_t off = 0;
  for (uint32_t b = 0; b < nb; ++b) {
    if (blk[b].crc_calc != blk[b].crc) return BZ_BLOCK_CRC;
    comb = ((comb << 1) | (comb >> 31)) ^ blk[b].crc;
    blk[b].out_off = off;
    off += blk[b].out_len;
  }
  if (comb != stored_comb) return BZ_STREAM_CRC;
  return off == dst_size ? R_OK : BZ_SIZE;
}

// ---------------------------------------------------------------- LZ4 frames
INF_HD uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
INF_HD uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

INF_HD uint32_t xxh32(const uint8_t* p, uint64_t n, uint32_t seed) {
  const uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
  uint64_t i = 0;
  uint32_t h;
  if (n >= 16) {
    uint32_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
    for (; i + 16 <= n; i += 16) {
      v1 = rotl32(v1 + rd32(p + i) * P2, 13) * P1;
      v2 = rotl32(v2 + rd32(p + i + 4) * P2, 13) * P1;
      v3 = rotl32(v3 + rd32(p + i + 8) * P2, 13) * P1;
      v4 = rotl32(v4 + rd32(p + i + 12) * P2, 13) * P1;
    }
    h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
  } else {
    h = seed + P5;
  }
  h += (uint32_t)n;
  for (; i + 4 <= n; i += 4) h = rotl32(h + rd32(p + i) * P3, 17) * P4;
  for (; i < n; ++i) h = rotl32(h + p[i] * P5, 11) * P1;
  h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
  return h;
}

// One LZ4 block src[0, n) decoded to dst at o (*o advanced); lo: the earliest byte a match may reach (the block's start
// for independent blocks, 0 for linked ones); lim: the end the block may write to.  Lane `ln` of `nl`.
INF_HD int32_t lz4_block(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t* o_io, uint64_t lo, uint64_t lim, int ln, int nl) {
  uint64_t i = 0, o = *o_io;
  for (;;) {
    if (i >= n) return LZ4_TRUNCATED;
    const uint32_t tok = src[i++];
    uint64_t lit = tok >> 4;
    if (lit == 15) {
      uint32_t v;
      do { if (i >= n) return LZ4_TRUNCATED; v = src[i++]; lit += v; } while (v == 255);
    }
    if (lit > n - i) return LZ4_TRUNCATED;
    if (lit > lim - o) return LZ4_OVERFLOW;
    for (uint64_t k = (uint64_t)ln; k < lit; k += (uint64_t)nl) dst[o + k] = src[i + k];
    i += lit; o += lit;
    if (i == n) break;                                    // the last sequence has literals only
    if (n - i < 2) return LZ4_TRUNCATED;
    const uint32_t off = (uint32_t)src[i] | (uint32_t)src[i + 1] << 8;
    i += 2;
    uint64_t ml = (tok & 15u) + 4;
    if ((tok & 15u) == 15) {
      uint32_t v;
      do { if (i >= n) return LZ4_TRUNCATED; v = src[i++]; ml += v; } while (v == 255);
    }
    if (off == 0 || off > o - lo) return LZ4_OFFSET;
    if (ml > lim - o) return LZ4_OVERFLOW;
    INF_SYNC();                                           // the match reads what earlier copies wrote
    const uint64_t from = o - off;
    for (uint64_t k = (uint64_t)ln; k < ml; k += (uint64_t)nl) dst[o + k] = dst[from + k % off];
    o += ml;
  }
  INF_SYNC();
  *o_io = o;
  return R_OK;
}

// One LZ4 frame src[0, n) -> dst[0, dst_size): exactly dst_size bytes or a refusal.
INF_HD int32_t lz4_frame(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t dst_size, int ln, int nl) {
  if (n < 4) return LZ4_MAGIC;
  const uint32_t magic = rd32(src);
  if (magic == 0x184C2102u) return LZ4_LEGACY;
  if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) return LZ4_SKIPPABLE;
  if (magic != 0x184D2204u) return LZ4_MAGIC;
  if (n < 7) return LZ4_TRUNCATED;
  const uint32_t flg = src[4], bd = src[5];
  if ((flg >> 6) != 1 || (flg & 2u) || (bd & 0x8Fu)) return LZ4_DESCRIPTOR;
  const int bmax_id = (int)(bd >> 4) & 7;
  if (bmax_id < 4) return LZ4_DESCRIPTOR;
  if (flg & 1u) return LZ4_DICT_ID;
  const bool indep = flg & 0x20u, bsum = flg & 0x10u, csize = flg & 8u, csum = flg & 4u;
  const uint64_t bmax = 1ull << (8 + 2 * bmax_id);
  uint64_t i = 6;
  if (csize) {
    if (n - i < 9) return LZ4_TRUNCATED;
    const uint64_t cs = (uint64_t)rd32(src + i) | (uint64_t)rd32(src + i + 4) << 32;
    i += 8;
    if (cs != dst_size) return LZ4_SIZE;
  }
  if (i >= n) return LZ4_TRUNCATED;
  if (((xxh32(src + 4, i - 4, 0) >> 8) & 0xFFu) != src[i]) return LZ4_HEADER_CHECKSUM;
  ++i;
  uint64_t o = 0;
  for (;;) {
    if (n - i < 4) return LZ4_TRUNCATED;
    const uint32_t w = rd32(src + i);
    i += 4;
    if (w == 0) break;                                    // end mark
    const uint64_t bs = w & 0x7FFFFFFFu;
    if (bs > bmax) return LZ4_BLOCK_SIZE;
    if (bs > n - i || (bsum && n - i - bs < 4)) return LZ4_TRUNCATED;
    if (bsum && xxh32(src + i, bs, 0) != rd32(src + i + bs)) return LZ4_BLOCK_CHECKSUM;
    const uint64_t lim = dst_size - o < bmax ? dst_size : o + bmax;
    if (w & 0x80000000u) {                                // stored uncompressed
      if (bs > lim - o) return LZ4_OVERFLOW;
      for (uint64_t k = (uint64_t)ln; k < bs; k += (uint64_t)nl) dst[o + k] = src[i + k];
      INF_SYNC();
      o += bs;
    } else {
      const int32_t r = lz4_block(src + i, bs, dst, &o, indep ? o : 0, lim, ln, nl);
      if (r) return r;
    }
    i += bs + (bsum ? 4 : 0);
  }
  if (csum) {
    if (n - i < 4) return LZ4_TRUNCATED;
    if (xxh32(dst, o, 0) != rd32(src + i)) return LZ4_CONTENT_CHECKSUM;
    i += 4;
  }
  if (i != n) return LZ4_TRAILING;
  return o == dst_size ? R_OK : LZ4_SIZE;
}

}  // namespace esvo_inflate
