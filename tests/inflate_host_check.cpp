// The chunk decoders of esvo_b200/csrc/inflate_core.h run on the host: every stage function inflate.cu launches, called in
// plain loops over blocks, tiles and samples (tests/test_inflate_core_host.py).
//   inflate_host_check <in.bin> <out.bin>
// in:  records  u32 codec (1 bz2, 2 LZ4) | u64 src_size | u64 dst_size | src bytes
// out: per record  i32 reason (0 = decoded) | dst_size bytes when the reason is 0
#include <cstdio>
#include <cstring>
#include <fstream>
#include <memory>
#include <vector>

#include "../esvo_b200/csrc/inflate_core.h"

using namespace esvo_inflate;

static int32_t bz2(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t dst_size) {
  static uint32_t tab[256];
  for (uint32_t i = 0; i < 256; ++i) tab[i] = crcEntry(i);
  const Bz2Caps cap = bz2Caps(dst_size);
  std::vector<uint32_t> tt(cap.tt + 1), hist((size_t)cap.tiles * 256 + 1), slen(cap.samp + 1), ssucc(cap.samp + 1), soff(cap.samp + 1);
  std::vector<uint8_t> pre(cap.tt + 1);
  std::vector<Bz2Block> blk(cap.nb);
  std::unique_ptr<Bz2State> st(new Bz2State);
  uint32_t nb = 0, comb = 0;
  int32_t r = bz2_parse(src, n, *st, tt.data(), cap, blk.data(), &nb, &comb);
  if (r) return r;
  for (uint32_t b = 0; b < nb; ++b) {
    const Bz2Block& B = blk[b];
    uint32_t* t = tt.data() + B.tt_off;
    uint32_t* h = hist.data() + (size_t)B.tile0 * 256;
    for (uint32_t k = 0; k < B.ntiles; ++k) {       // (b)
      std::memset(h + k * 256, 0, 1024);
      bz2_tile_count(t, k * kTile, std::min(B.nblock, (k + 1) * kTile), h + k * 256, 1);
    }
    uint32_t tot[256], base = 0;
    for (int s = 0; s < 256; ++s) tot[s] = bz2_scan_symbol(h, B.ntiles, s);
    for (int s = 0; s < 256; ++s) { bz2_scan_add(h, B.ntiles, s, base); base += tot[s]; }
    for (uint32_t k = 0; k < B.ntiles; ++k) bz2_tile_scatter(t, k * kTile, std::min(B.nblock, (k + 1) * kTile), h + k * 256, 1);
    uint32_t *l = slen.data() + B.samp0, *s = ssucc.data() + B.samp0, *o = soff.data() + B.samp0;   // (c)
    for (uint32_t j = 0; j < B.nsamp; ++j)
      if (!bz2_walk_len(t, B, j, l + j, s + j)) return BZ_BWT;
    if (!bz2_order(t, blk[b], l, s, o)) return BZ_BWT;
    for (uint32_t j = 0; j < B.nsamp; ++j)
      if (o[j] != kAbsentSample) bz2_walk_write(t, B, j, l[j], o[j], pre.data() + B.tt_off);
  }
  for (uint32_t b = 0; b < nb; ++b) {               // (d)
    const int64_t len = bz2_unrle(pre.data() + blk[b].tt_off, blk[b].nblock, nullptr, dst_size, tab, &blk[b].crc_calc);
    if (len < 0) return BZ_SIZE;
    blk[b].out_len = (uint32_t)len;
  }
  if ((r = bz2_finish(blk.data(), nb, comb, dst_size))) return r;
  for (uint32_t b = 0; b < nb; ++b) {
    uint32_t crc;
    bz2_unrle(pre.data() + blk[b].tt_off, blk[b].nblock, dst + blk[b].out_off, blk[b].out_len, tab, &crc);
  }
  return R_OK;
}

int main(int argc, char** argv) {
  if (argc != 3) { std::printf("usage: inflate_host_check <in.bin> <out.bin>\n"); return 64; }
  std::ifstream in(argv[1], std::ios::binary);
  std::ofstream out(argv[2], std::ios::binary);
  for (;;) {
    uint32_t codec; uint64_t n, m;
    if (!in.read((char*)&codec, 4)) break;
    in.read((char*)&n, 8); in.read((char*)&m, 8);
    std::vector<uint8_t> src(n), dst(m);       // exact sizes, so the sanitizers see any read or write outside them
    in.read((char*)src.data(), (std::streamsize)n);
    int32_t r = codec == 1 ? bz2(src.data(), n, dst.data(), m) : codec == 2 ? lz4_frame(src.data(), n, dst.data(), m, 0, 1) : R_CODEC;
    out.write((const char*)&r, 4);
    if (r == 0) out.write((const char*)dst.data(), (std::streamsize)m);
  }
  return 0;
}
