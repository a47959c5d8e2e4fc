// esvo_b200 product code -- device driver of the initialisation's semi-global block matching (sm_90a).
// The arithmetic lives in sgbm_core.h (per-work-item functions, pinned bit for bit against cv2 on the host by
// tests/test_sgbm_core_host.py); this file only maps work items to CUDA threads: one thread per image row (preparation,
// disparity selection), per matched pixel (costs, box sums, median) and per aggregation path (1 932 paths at 346x260).
// One-off at start-up (esvo_Mapping::InitializationAtTime, esvo_Mapping.cpp:433-492) -- not part of the per-frame hot path.
#include "common.cuh"
#include "sgbm_core.h"

namespace esvo {
using namespace esvo_sgbm;

__global__ void sgbm_prep_kernel(const uint8_t* left, const uint8_t* right, int pitch, Dims dm, int16_t* pl, int16_t* pr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * dm.H) return;
  const int y = t % dm.H;
  if (t < dm.H) prep_row(left, pitch, dm, y, pl + (size_t)y * 6 * dm.W);
  else prep_row(right, pitch, dm, y, pr + (size_t)y * 6 * dm.W);
}
__global__ void sgbm_pixcost_kernel(const int16_t* pl, const int16_t* pr, Dims dm, int16_t* pix) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= dm.H * dm.W1) return;
  const int y = t / dm.W1, x = t - y * dm.W1;
  pixel_cost(pl + (size_t)y * 6 * dm.W, pr + (size_t)y * 6 * dm.W, dm, x, pix + (size_t)t * dm.D);
}
__global__ void sgbm_boxh_kernel(const int16_t* pix, Dims dm, int16_t* hs) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= dm.H * dm.W1) return;
  const int y = t / dm.W1, x = t - y * dm.W1;
  box_h(pix + (size_t)y * dm.W1 * dm.D, dm, x, hs + (size_t)t * dm.D);
}
__global__ void sgbm_boxv_kernel(const int16_t* hs, Dims dm, int16_t* C) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= dm.H * dm.W1) return;
  const int y = t / dm.W1, x = t - y * dm.W1;
  box_v(hs, dm, y, x, C + (size_t)t * dm.D);
}
// path families, same enumeration as tests/sgbm_host_check.cpp:
//   [0,H) left->right rows | [H,2H) right->left rows | W1 columns top->down | W1 diagonals from the top edge going right-down |
//   W1 diagonals from the top edge going left-down | H-1 right-down diagonals from the left edge | H-1 left-down ones from the right edge
__global__ void sgbm_paths_kernel(const int16_t* C, Dims dm, int16_t* L0, int16_t* L1, int16_t* L2, int16_t* L3, int16_t* Lr) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int H = dm.H, W1 = dm.W1;
  if (t < H) { walk_path(C, L0, dm, 0, t, 1, 0); return; }
  t -= H;
  if (t < H) { walk_path(C, Lr, dm, W1 - 1, t, -1, 0); return; }
  t -= H;
  if (t < W1) { walk_path(C, L2, dm, t, 0, 0, 1); return; }
  t -= W1;
  if (t < W1) { walk_path(C, L1, dm, t, 0, 1, 1); return; }
  t -= W1;
  if (t < W1) { walk_path(C, L3, dm, t, 0, -1, 1); return; }
  t -= W1;
  if (t < H - 1) { walk_path(C, L1, dm, 0, t + 1, 1, 1); return; }
  t -= H - 1;
  if (t < H - 1) { walk_path(C, L3, dm, W1 - 1, t + 1, -1, 1); return; }
}
__global__ void sgbm_select_kernel(const int16_t* L0, const int16_t* L1, const int16_t* L2, const int16_t* L3, const int16_t* Lr, Dims dm,
                                   int32_t* scratch, int16_t* raw) {
  const int y = blockIdx.x * blockDim.x + threadIdx.x;
  if (y >= dm.H) return;
  select_row(L0, L1, L2, L3, Lr, dm, y, scratch + (size_t)y * 2 * dm.W, raw + (size_t)y * dm.W);
}
__global__ void sgbm_median_kernel(const int16_t* raw, Dims dm, int16_t* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= dm.H * dm.W) return;
  const int y = t / dm.W, x = t - y * dm.W;
  out[t] = median3(raw, dm, y, x);
}

// d_left / d_right: device images with row pitch `pitch`; d_out: H*W int16 on the device.
int sgbm_run(Ctx* c, const uint8_t* d_left, const uint8_t* d_right, int pitch, const Dims& dm, int16_t* d_out) {
  const size_t vol = (size_t)dm.H * dm.W1 * dm.D, rows = (size_t)dm.H * 6 * dm.W;
  int16_t *pl = nullptr, *pr = nullptr, *vols[8] = {nullptr}, *raw = nullptr;
  int32_t* scratch = nullptr;
  auto cleanup = [&]() { cudaFree(pl); cudaFree(pr); for (auto* v : vols) cudaFree(v); cudaFree(raw); cudaFree(scratch); };
  cudaError_t e = dmalloc(&pl, rows);
  if (e == cudaSuccess) e = dmalloc(&pr, rows);
  for (int k = 0; k < 8 && e == cudaSuccess; ++k) e = dmalloc(&vols[k], vol);
  if (e == cudaSuccess) e = dmalloc(&raw, (size_t)dm.H * dm.W);
  if (e == cudaSuccess) e = dmalloc(&scratch, (size_t)dm.H * 2 * dm.W);
  if (e != cudaSuccess) { cleanup(); c->set_error(cudaGetErrorString(e)); return ESVO_ERR_CUDA; }
  int16_t *pix = vols[0], *hs = vols[1], *C = vols[2], *L0 = vols[3], *L1 = vols[4], *L2 = vols[5], *L3 = vols[6], *Lr = vols[7];
  const int B = 64, npx = dm.H * dm.W1, npaths = 4 * dm.H + 3 * dm.W1 - 2;
  sgbm_prep_kernel<<<div_up(2 * dm.H, B), B, 0, c->stream>>>(d_left, d_right, pitch, dm, pl, pr);
  sgbm_pixcost_kernel<<<div_up(npx, B), B, 0, c->stream>>>(pl, pr, dm, pix);
  sgbm_boxh_kernel<<<div_up(npx, B), B, 0, c->stream>>>(pix, dm, hs);
  sgbm_boxv_kernel<<<div_up(npx, B), B, 0, c->stream>>>(hs, dm, C);
  sgbm_paths_kernel<<<div_up(npaths, B), B, 0, c->stream>>>(C, dm, L0, L1, L2, L3, Lr);
  sgbm_select_kernel<<<div_up(dm.H, 32), 32, 0, c->stream>>>(L0, L1, L2, L3, Lr, dm, scratch, raw);
  sgbm_median_kernel<<<div_up(dm.H * dm.W, 256), 256, 0, c->stream>>>(raw, dm, d_out);
  c->launches += 7;
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  cleanup();
  if (e != cudaSuccess) { c->set_error(cudaGetErrorString(e)); return ESVO_ERR_CUDA; }
  return ESVO_OK;
}

}  // namespace esvo
