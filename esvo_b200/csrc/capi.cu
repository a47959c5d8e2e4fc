// esvo_b200 product code -- C ABI (include/esvo_b200.h) over the CUDA stages.
// Host logic only: argument checks, buffer management, H2D/D2H staging and kernel sequencing.
// There is no CPU fallback: every entry point that computes does so with the kernels in this
// directory, and esvo_create fails when no CUDA device is usable.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace esvo {

// 5x5 Gaussian on u8 (cv::GaussianBlur sigma=0: [1 4 6 4 1]/16 per axis, fixed point, round half
// up, BORDER_REFLECT_101) -- TimeSurfaceObservation::GaussianBlurTS / getTimeSurfaceNegative.
__device__ __forceinline__ int refl101(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
  return p;
}
__global__ void gauss5_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int W, int H, int pitch) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const int k[5] = {1, 4, 6, 4, 1};
  int s = 0;
#pragma unroll
  for (int dy = -2; dy <= 2; ++dy) {
    const uint8_t* row = src + (size_t)refl101(y + dy, H) * pitch;
    int r = 0;
#pragma unroll
    for (int dx = -2; dx <= 2; ++dx) r += k[dx + 2] * row[refl101(x + dx, W)];
    s += k[dy + 2] * r;
  }
  dst[(size_t)y * pitch + x] = (uint8_t)((s + 128) >> 8);
}

__global__ void fp64_probe_kernel(double* out, int iters) {
  double a = threadIdx.x * 1e-3 + 1.0, b = 1.000001, cc = 0.5, d = a + 1;
  for (int i = 0; i < iters; ++i) { a = fma(a, b, cc); d = fma(d, b, cc); }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a + d;
}

int smooth_obs(Ctx* c) {
  SlotBufs& f = c->slot();
  dim3 b(32, 8), g(div_up(c->dc.W, 32), div_up(c->dc.H, 8));
  f.obs_ls = f.own_ls; f.obs_rs = f.own_rs;
  gauss5_u8_kernel<<<g, b, 0, c->stream>>>(f.obs_l, f.obs_ls, c->dc.W, c->dc.H, c->dc.pitch);
  gauss5_u8_kernel<<<g, b, 0, c->stream>>>(f.obs_r, f.obs_rs, c->dc.W, c->dc.H, c->dc.pitch);
  c->launches += 2;
  return ESVO_OK;
}

int map_alloc_inputs(Ctx* c, size_t n_ev, size_t n_poses) {
  SlotBufs& f = c->slot();
  if (n_ev > f.ev_cap) {
    size_t cap = std::max<size_t>(n_ev, 1024);
    void* olds[] = {f.bm.flag, f.bm.disp, f.bm.pose_idx, f.bm.cost, f.bm.xrect,
                    f.d_seeds, f.lm_flag, f.lm_res, f.d_pts};
    for (void* p : olds) if (p) cudaFree(p);
    ESVO_CUDA_TRY(c, dmalloc(&f.bm.flag, cap)); ESVO_CUDA_TRY(c, dmalloc(&f.bm.disp, cap));
    ESVO_CUDA_TRY(c, dmalloc(&f.bm.pose_idx, cap)); ESVO_CUDA_TRY(c, dmalloc(&f.bm.cost, cap));
    ESVO_CUDA_TRY(c, dmalloc(&f.bm.xrect, 2 * cap)); ESVO_CUDA_TRY(c, dmalloc(&f.d_seeds, cap));
    ESVO_CUDA_TRY(c, dmalloc(&f.lm_flag, cap)); ESVO_CUDA_TRY(c, dmalloc(&f.lm_res, 3 * cap));
    ESVO_CUDA_TRY(c, dmalloc(&f.d_pts, cap));
    f.ev_cap = cap;
  }
  if (n_poses > f.pose_cap) f.pose_cap = std::max<size_t>(n_poses, 256);
  const size_t need = f.ev_cap * 12 + f.pose_cap * 136 + 64;
  if (need > f.in_bytes) {
    if (f.ev_in_valid) { ESVO_CUDA_TRY(c, cudaEventSynchronize(f.ev_in)); f.ev_in_valid = false; }
    if (f.d_in) { ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream)); cudaFree(f.d_in); }
    if (f.h_in) cudaFreeHost(f.h_in);
    ESVO_CUDA_TRY(c, dmalloc(&f.d_in, need));
    ESVO_CUDA_TRY(c, cudaMallocHost((void**)&f.h_in, need));
    if (!f.ev_in) ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&f.ev_in, cudaEventDisableTiming));
    f.in_bytes = need;
    f.d_ex = f.d_ey = nullptr; f.d_et = f.d_pose_t = nullptr; f.d_poses = nullptr;
  }
  return ESVO_OK;
}

// Host arrays -> the slot's packed device block with ONE H2D copy (layout: et | pose_t | poses | ex | ey).
int stage_inputs_packed(Ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et, size_t n, const int64_t* pt,
                        const double* poses, size_t np) {
  int rc = map_alloc_inputs(c, n, np);
  if (rc) return rc;
  SlotBufs& f = c->slot();
  f.n_ev = n; f.n_poses = np;
  if (f.ev_in_valid) ESVO_CUDA_TRY(c, cudaEventSynchronize(f.ev_in));   // the previous upload from this pinned mirror (long done)
  const size_t o_et = 0, o_pt = o_et + n * 8, o_ps = o_pt + np * 8, o_ex = o_ps + np * 128, o_ey = o_ex + ((n * 2 + 7) & ~(size_t)7);
  const size_t total = o_ey + n * 2;
  if (n) { std::memcpy(f.h_in + o_et, et, n * 8); std::memcpy(f.h_in + o_ex, ex, n * 2); std::memcpy(f.h_in + o_ey, ey, n * 2); }
  if (np) { std::memcpy(f.h_in + o_pt, pt, np * 8); std::memcpy(f.h_in + o_ps, poses, np * 128); }
  f.d_et = (int64_t*)(f.d_in + o_et); f.d_pose_t = (int64_t*)(f.d_in + o_pt); f.d_poses = (double*)(f.d_in + o_ps);
  f.d_ex = (uint16_t*)(f.d_in + o_ex); f.d_ey = (uint16_t*)(f.d_in + o_ey);
  if (total) {
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.d_in, f.h_in, total, cudaMemcpyHostToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaEventRecord(f.ev_in, c->stream));
    f.ev_in_valid = true;
  }
  return ESVO_OK;
}

static int slot_alloc(Ctx* c, int i) {
  SlotBufs& s = c->slots[i];
  if (s.allocated) return ESVO_OK;
  const size_t nimg = (size_t)c->dc.pitch * c->dc.H;
  if (!s.stream) ESVO_CUDA_TRY(c, cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
  ESVO_CUDA_TRY(c, dmalloc(&s.obs_l, nimg)); ESVO_CUDA_TRY(c, dmalloc(&s.obs_r, nimg));
  ESVO_CUDA_TRY(c, dmalloc(&s.own_ls, nimg)); ESVO_CUDA_TRY(c, dmalloc(&s.own_rs, nimg));
  s.obs_ls = s.own_ls; s.obs_rs = s.own_rs;
  ESVO_CUDA_TRY(c, dmalloc(&s.d_counters, kCounters));
  ESVO_CUDA_TRY(c, cudaMallocHost((void**)&s.h_counters, kCounters * 8));
  ESVO_CUDA_TRY(c, cudaMemset(s.d_counters, 0, kCounters * 8));
  ESVO_CUDA_TRY(c, cudaMemset(s.obs_l, 0, nimg)); ESVO_CUDA_TRY(c, cudaMemset(s.obs_r, 0, nimg));
  ESVO_CUDA_TRY(c, cudaMemset(s.own_ls, 0, nimg)); ESVO_CUDA_TRY(c, cudaMemset(s.own_rs, 0, nimg));
  ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&s.ev_obs, cudaEventDisableTiming));
  ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&s.ev_free, cudaEventDisableTiming));
  ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&s.ev_pts, cudaEventDisableTiming));
  ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&s.ev_fuse, cudaEventDisableTiming));
  if (int rc = fuse_alloc(c, &s.map)) return rc;   // the slot's own map / fusion staging
  s.allocated = true;
  return ESVO_OK;
}
// Releases everything slot i holds, allocated or partly allocated (the ctx is drained).
static void slot_free(Ctx* c, int i) {
  SlotBufs& s = c->slots[i];
  fuse_free(s.map);
  s.map = nullptr;
  void* ps[] = {s.obs_l, s.obs_r, s.own_ls, s.own_rs, s.d_counters, s.d_in, s.bm.flag, s.bm.disp, s.bm.pose_idx, s.bm.cost, s.bm.xrect, s.d_seeds, s.lm_flag, s.lm_res,
                s.d_pts};
  for (void* p : ps) if (p) cudaFree(p);
  if (s.h_counters) cudaFreeHost(s.h_counters);
  if (s.h_in) cudaFreeHost(s.h_in);
  if (s.ev_in) cudaEventDestroy(s.ev_in);
  if (s.ev_obs) cudaEventDestroy(s.ev_obs);
  if (s.ev_free) cudaEventDestroy(s.ev_free);
  if (s.ev_pts) cudaEventDestroy(s.ev_pts);
  if (s.ev_fuse) cudaEventDestroy(s.ev_fuse);
  if (s.ev_dl) cudaEventDestroy(s.ev_dl);
  if (s.d_dl) cudaFree(s.d_dl);
  if (s.d_dl_keys) cudaFree(s.d_dl_keys);
  if (s.d_dlscal) cudaFree(s.d_dlscal);
  if (s.h_dlscal) cudaFreeHost(s.h_dlscal);
  if (s.h_dl) cudaFreeHost(s.h_dl);
  if (s.stream && s.stream != c->s_main) cudaStreamDestroy(s.stream);
}
int drain(Ctx* c) {
  for (int k = 0; k < 2; ++k) if (c->s_tsc[k]) ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->s_tsc[k]));
  for (int i = 0; i < kMaxSlots; ++i) {
    if (c->slots[i].stream) ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->slots[i].stream));
  }
  if (c->s_copy) ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->s_copy));
  // Everything pushed so far has landed: refresh the host's view of the newest stamp from the device scalar, so that
  // builds after device-resident pushes can take the short path again (ts.cu: maybe_general)
  for (int k = 0; k < 2; ++k) {
    TsState& t = c->ts[k];
    if (!t.host_knows && !t.unordered && t.max_t) {
      long long v = 0;
      ESVO_CUDA_TRY(c, cudaMemcpy(&v, t.max_t, 8, cudaMemcpyDeviceToHost));
      t.host_max_t = v; t.host_knows = true;
    }
  }
  return ESVO_OK;
}

static int upload_tables(Ctx* c) {
  const size_t npix = (size_t)c->dc.W * c->dc.H;
  ESVO_CUDA_TRY(c, cudaMemcpy(c->d_lut, c->cam[0].lut.data(), 2 * npix * 8, cudaMemcpyHostToDevice));
  ESVO_CUDA_TRY(c, cudaMemcpy(c->d_mask, c->cam[0].mask.data(), npix, cudaMemcpyHostToDevice));
  for (int cam = 0; cam < 2; ++cam) {
    ESVO_CUDA_TRY(c, cudaMemcpy(c->ts[cam].map1, c->cam[cam].map1.data(), npix * 4, cudaMemcpyHostToDevice));
    ESVO_CUDA_TRY(c, cudaMemcpy(c->ts[cam].map2, c->cam[cam].map2.data(), npix * 4, cudaMemcpyHostToDevice));
  }
  return ESVO_OK;
}

// The part of esvo_set_ts_pair behind the image copies: the observation pose, and the raw pair as the solver's view of it until
// createMatchProblem smooths it.
static int obs_set_pose(Ctx* c, const double T[16]) {
  SlotBufs& f = c->slot();
  const size_t nimg = (size_t)c->dc.pitch * c->dc.H;
  std::memcpy(f.T_world_left, T, sizeof(f.T_world_left));
  rigid_inverse(T, f.T_left_world_inv);
  if (!c->prm.smooth_time_surface) { f.obs_ls = f.obs_l; f.obs_rs = f.obs_r; }
  else {
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.obs_ls, f.obs_l, nimg, cudaMemcpyDeviceToDevice, c->stream));
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.obs_rs, f.obs_r, nimg, cudaMemcpyDeviceToDevice, c->stream));
  }
  ESVO_CUDA_TRY(c, cudaEventRecord(f.ev_obs, c->stream));
  c->obs_set = true;
  return ESVO_OK;
}

int fetch_counters(Ctx* c) {
  SlotBufs& f = c->slot();
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.h_counters, f.d_counters, kCounters * 8, cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  return ESVO_OK;
}

}  // namespace esvo

using namespace esvo;

extern "C" {

ESVO_API void esvo_default_params(esvo_params* p) { host_default_params(p); }
ESVO_API const char* esvo_version(void) { return "esvo_b200 0.1 (sm_90a)"; }
ESVO_API const char* esvo_last_error(esvo_ctx* c) { return c ? c->err.c_str() : "null ctx"; }
ESVO_API void* esvo_stream(esvo_ctx* c) { return c ? (void*)c->stream : nullptr; }
ESVO_API uint64_t esvo_launch_count(esvo_ctx* c) { return c ? c->launches : 0; }
ESVO_API int esvo_sync(esvo_ctx* c) { CHECK_CTX(c); return drain(c); }
// Measured FP64 FMA rate of this GPU (bench.py: the denominator of the fp64 roofline): SMs*8 blocks x 256 threads, two
// independent dependent-FMA chains per thread, CUDA-event timed on the ctx stream.  Returns TFLOP/s (2 flops per FMA).
ESVO_API int esvo_debug_fp64_probe(esvo_ctx* c, double* tflops_out) {
  CHECK_CTX(c);
  if (!tflops_out) return ESVO_ERR_INVALID_ARG;
  int rc = drain(c);
  if (rc) return rc;
  const int blocks = c->num_sms * 8, threads = 256, iters = 20000;
  double* out = nullptr;
  ESVO_CUDA_TRY(c, dmalloc(&out, (size_t)blocks * threads));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  fp64_probe_kernel<<<blocks, threads, 0, c->stream>>>(out, 64);
  float best = 1e30f;
  for (int rep = 0; rep < 3; ++rep) {
    cudaEventRecord(e0, c->stream);
    fp64_probe_kernel<<<blocks, threads, 0, c->stream>>>(out, iters);
    cudaEventRecord(e1, c->stream);
    cudaEventSynchronize(e1);
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    best = std::min(best, ms);
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(out);
  ESVO_CUDA_TRY(c, cudaGetLastError());
  *tflops_out = 2.0 * 2.0 * iters * (double)blocks * threads / (best * 1e-3) / 1e12;
  return ESVO_OK;
}
ESVO_API int esvo_set_pipeline_depth(esvo_ctx* c, int depth) {
  CHECK_CTX(c);
  if (depth < 1 || depth > kMaxSlots) return ESVO_ERR_INVALID_ARG;
  int rc = drain(c);
  if (rc) return rc;
  if (depth > 1) {
    // The time-surface chain of a frame is ~8 short dependent kernels per camera; with the SMs saturated by the
    // LM kernels of the frames in flight, each of them would queue behind pending LM blocks.  The two cameras get
    // their own streams, at the highest priority: their blocks are placed as soon as any LM block retires.
    int lo = 0, hi = 0;
    ESVO_CUDA_TRY(c, cudaDeviceGetStreamPriorityRange(&lo, &hi));
    for (int k = 0; k < 2; ++k)
      if (c->s_tsc[k] == c->s_main) ESVO_CUDA_TRY(c, cudaStreamCreateWithPriority(&c->s_tsc[k], cudaStreamNonBlocking, hi));
    if (!c->ev_ts_join) ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&c->ev_ts_join, cudaEventDisableTiming));
    for (int i = 1; i < depth; ++i) if ((rc = slot_alloc(c, i))) return rc;
  } else {
    for (int k = 0; k < 2; ++k) if (c->s_tsc[k] != c->s_main) { cudaStreamDestroy(c->s_tsc[k]); c->s_tsc[k] = c->s_main; }
  }
  c->depth = depth;
  c->frame_no = 0;
  c->activate(0);
  return ESVO_OK;
}

ESVO_API esvo_ctx* esvo_create(int device, const esvo_calib* left, const esvo_calib* right, const esvo_params* p,
                               int* status_out) {
  auto fail = [&](int code) -> esvo_ctx* { if (status_out) *status_out = code; return nullptr; };
  if (!left || !right || !p || left->width != right->width || left->height != right->height || left->width <= 0 ||
      left->height <= 0)
    return fail(ESVO_ERR_INVALID_ARG);
  if (p->patch_size_x * p->patch_size_y > kMaxPatch || p->patch_size_x < 1 || p->patch_size_y < 1 ||
      !(p->patch_size_x & 1) || !(p->patch_size_y & 1))
    return fail(ESVO_ERR_UNSUPPORTED);
  // A negative regularisation radius is an empty neighbourhood loop in DepthRegularization::apply, but the warp form's
  // (2r+1)^2 window would read pixel (row+1, col+1): refused rather than given a second meaning.
  if (p->reg_radius < 0) return fail(ESVO_ERR_UNSUPPORTED);
  // The closed-form cam2World / propagation (lm.cu, fuse.cu) assume a canonical rectified projection
  // P = [fx 0 cx tx; 0 fy cy ty; 0 0 1 0] (every shipped calibration); the reference's 4x4 inverse is more general.
  for (const esvo_calib* cal : {left, right})
    if (cal->P[1] != 0 || cal->P[4] != 0 || cal->P[8] != 0 || cal->P[9] != 0 || cal->P[10] != 1 || cal->P[11] != 0)
      return fail(ESVO_ERR_UNSUPPORTED);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return fail(ESVO_ERR_NO_DEVICE);
  if (cudaSetDevice(device) != cudaSuccess) return fail(ESVO_ERR_NO_DEVICE);
  esvo_ctx* c = new esvo_ctx();
  c->device = device;
  if (cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) { delete c; return fail(ESVO_ERR_CUDA); }
  c->prm = *p;
  host_camera_init(c->cam[0], *left);
  host_camera_init(c->cam[1], *right);
  DevConsts& d = c->dc;
  d.W = left->width; d.H = left->height; d.pitch = (d.W + 15) / 16 * 16;
  d.wx = p->patch_size_x; d.wy = p->patch_size_y;
  d.baseline = host_baseline(c->cam[1]);
  {  // esvo_Mapping.cpp:110-116
    double f = (c->cam[0].P[0] + c->cam[0].P[5]) / 2, b = d.baseline;
    size_t minD = std::max(size_t(std::floor(f * b * p->invdepth_min_range)), (size_t)0);
    size_t maxD = size_t(std::ceil(f * b * p->invdepth_max_range));
    d.dmin = (int)std::max(minD, (size_t)p->bm_min_disparity);
    d.dmax = (int)std::min(maxD, (size_t)p->bm_max_disparity);
  }
  d.step = std::max(1, p->bm_step); d.updown = p->bm_updown; d.zncc_thr = p->bm_zncc_threshold;
  d.fx = c->cam[0].P[0]; d.fy = c->cam[0].P[5]; d.cx = c->cam[0].P[2]; d.cy = c->cam[0].P[6];
  std::memcpy(d.Pl, c->cam[0].P, sizeof(d.Pl)); std::memcpy(d.Pr, c->cam[1].P, sizeof(d.Pr));
  d.lsnorm = p->lsnorm; d.max_iter = p->max_iteration; d.td_nu = p->td_nu; d.td_scale = p->td_scale;
  d.td_scale2 = p->td_scale * p->td_scale;
  d.td_stdvar = std::sqrt(p->td_nu / (p->td_nu - 2) * d.td_scale2);  // DepthProblem.h:34
  d.NT = std::max(1, p->num_thread_mapping);
  if (d.dmax >= d.dmin && (d.dmax - d.dmin) / d.step + 1 > 192 && d.step > 1) { delete c; return fail(ESVO_ERR_UNSUPPORTED); }
  auto bail = [&](int code) -> esvo_ctx* { esvo_destroy(c); return fail(code); };
  if (cudaStreamCreateWithFlags(&c->s_main, cudaStreamNonBlocking) != cudaSuccess) return bail(ESVO_ERR_CUDA);
  c->stream = c->s_tsc[0] = c->s_tsc[1] = c->s_main;
  c->slots[0].stream = c->s_main;
  const size_t npix = (size_t)d.W * d.H;
  if (slot_alloc(c, 0)) return bail(ESVO_ERR_CUDA);
  if (dmalloc(&c->d_lut, 2 * npix) || dmalloc(&c->d_mask, npix)) return bail(ESVO_ERR_CUDA);
  for (int cam = 0; cam < 2; ++cam) if (ts_alloc(c, cam)) return bail(ESVO_ERR_CUDA);
  if (upload_tables(c)) return bail(ESVO_ERR_CUDA);
  if (map_alloc_inputs(c, 16384, 512)) return bail(ESVO_ERR_CUDA);
  if (track_alloc(c)) return bail(ESVO_ERR_CUDA);
  if (status_out) *status_out = ESVO_OK;
  return c;
}

ESVO_API void esvo_destroy(esvo_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  drain(c);
  c->stream = c->s_main;
  for (int cam = 0; cam < 2; ++cam) ts_free(c, cam);
  track_free(c);
  ew_free(c);
  if (c->d_lut) cudaFree(c->d_lut);
  if (c->d_mask) cudaFree(c->d_mask);
  for (int i = 0; i < kMaxSlots; ++i) slot_free(c, i);
  for (auto& f : c->win) { cudaFree(f.pts); cudaFree(f.cnt); if (f.last_read) cudaEventDestroy(f.last_read); }
  for (auto& f : c->win_pool) { cudaFree(f.pts); cudaFree(f.cnt); if (f.last_read) cudaEventDestroy(f.last_read); }
  for (auto e : c->prof_pool) cudaEventDestroy(e);
  if (c->hist.buf) cudaFree(c->hist.buf);
  for (auto e : c->hist.ev) cudaEventDestroy(e);
  if (c->hist.ev_join) cudaEventDestroy(c->hist.ev_join);
  for (void* p : {(void*)c->pub.xyz, (void*)c->pub.sorted, (void*)c->pub.d_scal}) if (p) cudaFree(p);
  if (c->pub.h_scal) cudaFreeHost(c->pub.h_scal);
  for (int k = 0; k < 2; ++k) if (c->s_tsc[k] && c->s_tsc[k] != c->s_main) cudaStreamDestroy(c->s_tsc[k]);
  if (c->ev_ts_join) cudaEventDestroy(c->ev_ts_join);
  if (c->s_copy) cudaStreamDestroy(c->s_copy);
  if (c->s_main) cudaStreamDestroy(c->s_main);
  delete c;
}

ESVO_API int esvo_set_rectify_tables(esvo_ctx* c, int cam, const float* m1, const float* m2, const double* lut,
                                     const uint8_t* mask) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  const size_t n = (size_t)c->dc.W * c->dc.H;
  if (m1) c->cam[cam].map1.assign(m1, m1 + n);
  if (m2) c->cam[cam].map2.assign(m2, m2 + n);
  if (lut) c->cam[cam].lut.assign(lut, lut + 2 * n);
  c->tables_version++;
  if (mask) c->cam[cam].mask.assign(mask, mask + n);
  { int rc0 = drain(c); if (rc0) return rc0; }   // kernels of other pipeline slots / the TS streams may still read the tables
  return upload_tables(c);
}
ESVO_API int esvo_get_rectify_tables(esvo_ctx* c, int cam, float* m1, float* m2, double* lut, uint8_t* mask) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  const size_t n = (size_t)c->dc.W * c->dc.H;
  if (m1) std::memcpy(m1, c->cam[cam].map1.data(), n * 4);
  if (m2) std::memcpy(m2, c->cam[cam].map2.data(), n * 4);
  if (lut) std::memcpy(lut, c->cam[cam].lut.data(), 2 * n * 8);
  if (mask) std::memcpy(mask, c->cam[cam].mask.data(), n);
  return ESVO_OK;
}
ESVO_API int esvo_compute_rectify_tables(const esvo_calib* cal, float* m1, float* m2, double* lut, uint8_t* mask) {
  if (!cal || cal->width <= 0 || cal->height <= 0) return ESVO_ERR_INVALID_ARG;
  HostCamera hc;
  host_camera_init(hc, *cal);
  const size_t n = (size_t)hc.W * hc.H;
  if (m1) std::memcpy(m1, hc.map1.data(), n * 4);
  if (m2) std::memcpy(m2, hc.map2.data(), n * 4);
  if (lut) std::memcpy(lut, hc.lut.data(), 2 * n * 8);
  if (mask) std::memcpy(mask, hc.mask.data(), n);
  return ESVO_OK;
}
ESVO_API int esvo_get_derived(esvo_ctx* c, double out[4]) {
  CHECK_CTX(c);
  out[0] = c->dc.baseline; out[1] = c->dc.dmin; out[2] = c->dc.dmax; out[3] = c->dc.td_stdvar;
  return ESVO_OK;
}

// ---------------- time surface ----------------
ESVO_API int esvo_stage_ts_events(esvo_ctx* c, int cam, const uint16_t* x, const uint16_t* y, const int64_t* t,
                                  const uint8_t* pol, size_t n) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || (n && (!x || !y || !t))) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return ts_push(c, cam, x, y, t, pol, n, false);
}
ESVO_API int esvo_ts_push_events_dev(esvo_ctx* c, int cam, const uint16_t* x, const uint16_t* y, const int64_t* t,
                                     const uint8_t* pol, size_t n) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || (n && (!x || !y || !t))) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return ts_push(c, cam, x, y, t, pol, n, true);
}
ESVO_API int esvo_ts_push_events(esvo_ctx* c, int cam, const uint16_t* x, const uint16_t* y, const int64_t* t,
                                 const uint8_t* pol, size_t n) {
  int rc = esvo_stage_ts_events(c, cam, x, y, t, pol, n);
  if (rc) return rc;
  // the caller's buffers may be reused as soon as we return
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->s_tsc[cam]));
  return ESVO_OK;
}
ESVO_API int esvo_ts_push_event_array(esvo_ctx* c, int cam, const uint8_t* const* runs, const size_t* n_events, int n_runs) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || n_runs < 0 || (n_runs && (!runs || !n_events))) return ESVO_ERR_INVALID_ARG;
  for (int k = 0; k < n_runs; ++k) if (n_events[k] && !runs[k]) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return ts_push_packed_host(c, cam, runs, n_events, n_runs);
}
ESVO_API int esvo_ts_push_event_array_dev(esvo_ctx* c, int cam, const uint8_t* packed_dev, size_t n) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || (n && !packed_dev)) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return ts_push_packed(c, cam, packed_dev, n, nullptr);
}
ESVO_API int esvo_ts_events_pushed(esvo_ctx* c, int cam, int64_t* total) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || !total) return ESVO_ERR_INVALID_ARG;
  *total = c->ts[cam].log_base + (int64_t)c->ts[cam].log_n;
  return ESVO_OK;
}
// ---------------- hot pixels (hotpix.cu) ----------------
ESVO_API int esvo_hotpix_count_event_array(esvo_ctx* c, int cam, const uint8_t* const* runs, const size_t* n_events, int n_runs) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || n_runs < 0 || (n_runs && (!runs || !n_events))) return ESVO_ERR_INVALID_ARG;
  for (int k = 0; k < n_runs; ++k) if (n_events[k] && !runs[k]) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return hp_count_packed_host(c, cam, runs, n_events, n_runs);
}
ESVO_API int esvo_hotpix_count_event_array_dev(esvo_ctx* c, int cam, const uint8_t* packed_dev, size_t n) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1 || (n && !packed_dev)) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return hp_count_packed(c, cam, packed_dev, n);
}
ESVO_API int esvo_hotpix_select(esvo_ctx* c, int cam, double k, int64_t* n_hot) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return hp_select(c, cam, k, n_hot);
}
ESVO_API int esvo_hotpix_read(esvo_ctx* c, int cam, uint32_t* counts, uint8_t* mask) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return hp_read(c, cam, counts, mask);
}
ESVO_API int esvo_hotpix_clear(esvo_ctx* c, int cam) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return hp_clear(c, cam);
}
ESVO_API int esvo_run_ts_build(esvo_ctx* c, int cam, int64_t T) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  StreamScope sc(c, c->s_tsc[cam]);
  return ts_run_build(c, cam, T);
}
ESVO_API int esvo_ts_build(esvo_ctx* c, int cam, int64_t T, int64_t* idx_out, uint8_t* ts_out) {
  int rc = esvo_run_ts_build(c, cam, T);
  if (rc) return rc;
  TsState& s = c->ts[cam];
  const DevConsts& d = c->dc;
  StreamScope sc(c, c->s_tsc[cam]);
  if (idx_out) ESVO_CUDA_TRY(c, cudaMemcpyAsync(idx_out, s.out_idx, (size_t)d.W * d.H * 8, cudaMemcpyDeviceToHost, c->stream));
  if (ts_out) ESVO_CUDA_TRY(c, cudaMemcpy2DAsync(ts_out, d.W, s.img_out, d.pitch, d.W, d.H, cudaMemcpyDeviceToHost, c->stream));
  int32_t flags[12] = {0};
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(flags, s.scalars, sizeof(flags), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (flags[1]) { c->set_error("events were not pushed in time order (unsupported on the device path)"); return ESVO_ERR_UNSUPPORTED; }
  long long fold_t;                                      // stamp of the newest event folded out of the resident log (ts_make_room)
  std::memcpy(&fold_t, flags + 10, 8);
  if (s.log_base > 0 && (long long)T <= fold_t) {
    c->set_error("t_sync " + std::to_string((long long)T) + " is not newer than the events folded out of the resident log; the oldest answerable t_sync is " +
                 std::to_string(fold_t + 1));
    return ESVO_ERR_UNSUPPORTED;
  }
  return ESVO_OK;
}
ESVO_API int esvo_ts_set_unordered_input(esvo_ctx* c, int cam, int enable) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  TsState& s = c->ts[cam];
  // the scan carries events_.back() from push to push; ordered pushes do not record it, so the switch cannot be turned on over them
  if (enable && !s.unordered && (s.log_n || s.log_base)) {
    c->set_error("esvo_ts_set_unordered_input: the camera already holds events pushed as ordered input; call esvo_ts_reset first");
    return ESVO_ERR_UNSUPPORTED;
  }
  s.unordered = enable != 0;
  return ESVO_OK;
}
ESVO_API int esvo_ts_reset(esvo_ctx* c, int cam) {
  CHECK_CTX(c);
  if (cam < 0 || cam > 1) return ESVO_ERR_INVALID_ARG;
  int rc = drain(c);
  if (rc) return rc;
  StreamScope sc(c, c->s_tsc[cam]);
  return ts_reset_state(c, cam);
}

// ---------------- mapping ----------------
ESVO_API int esvo_set_ts_pair(esvo_ctx* c, const uint8_t* l, const uint8_t* r, const double T[16]) {
  CHECK_CTX(c);
  if (!T) return ESVO_ERR_INVALID_ARG;
  { int rc0 = drain(c); if (rc0) return rc0; }
  SlotBufs& f = c->slot();
  const DevConsts& d = c->dc;
  const size_t nimg = (size_t)d.pitch * d.H;
  if (l) ESVO_CUDA_TRY(c, cudaMemcpy2DAsync(f.obs_l, d.pitch, l, d.W, d.W, d.H, cudaMemcpyHostToDevice, c->stream));
  else {
    if (!c->ts[0].built) { c->set_error("ts_left == NULL but no time surface was built for camera 0"); return ESVO_ERR_STATE; }
    if (f.obs_l != c->ts[0].last_img) ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.obs_l, c->ts[0].last_img, nimg, cudaMemcpyDeviceToDevice, c->stream));
  }
  if (r) ESVO_CUDA_TRY(c, cudaMemcpy2DAsync(f.obs_r, d.pitch, r, d.W, d.W, d.H, cudaMemcpyHostToDevice, c->stream));
  else {
    if (!c->ts[1].built) { c->set_error("ts_right == NULL but no time surface was built for camera 1"); return ESVO_ERR_STATE; }
    if (f.obs_r != c->ts[1].last_img) ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.obs_r, c->ts[1].last_img, nimg, cudaMemcpyDeviceToDevice, c->stream));
  }
  int rc = obs_set_pose(c, T);
  if (rc) return rc;
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // the caller's images are host memory
  return ESVO_OK;
}

// ---- time-surface history (TimeSurfaceHistory, esvo_Mapping.h: std::map<ros::Time, TimeSurfaceObservation>) ----
ESVO_API int esvo_ts_history_reserve_dev(esvo_ctx* c, size_t capacity) {
  CHECK_CTX(c);
  { int rc0 = drain(c); if (rc0) return rc0; }
  Ctx::TsHistory& h = c->hist;
  if (h.buf) { cudaFree(h.buf); h.buf = nullptr; }
  for (auto e : h.ev) cudaEventDestroy(e);
  h.stamp.clear(); h.used.clear(); h.ev.clear();
  if (capacity == 0) return ESVO_OK;
  const size_t nimg = (size_t)c->dc.pitch * c->dc.H;
  ESVO_CUDA_TRY(c, dmalloc(&h.buf, 2 * capacity * nimg));
  if (!h.ev_join) ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&h.ev_join, cudaEventDisableTiming));
  h.stamp.assign(capacity, 0); h.used.assign(capacity, false); h.ev.assign(capacity, nullptr);
  for (auto& e : h.ev) ESVO_CUDA_TRY(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  return ESVO_OK;
}
ESVO_API int esvo_ts_history_store_dev(esvo_ctx* c, int64_t stamp) {
  CHECK_CTX(c);
  Ctx::TsHistory& h = c->hist;
  if (!h.cap()) { c->set_error("esvo_ts_history_store_dev: no history reserved (esvo_ts_history_reserve_dev)"); return ESVO_ERR_STATE; }
  if (!c->ts[0].built || !c->ts[1].built) { c->set_error("esvo_ts_history_store_dev needs a built time surface for both cameras"); return ESVO_ERR_STATE; }
  // operator[] then erase(begin()) while over capacity: a stored stamp is overwritten, a new one takes a free entry or the
  // one with the smallest stamp -- unless it is itself the smallest, which the map would insert and drop again at once
  size_t i = h.cap(), oldest = h.cap();
  for (size_t k = 0; k < h.cap() && i == h.cap(); ++k) if (h.used[k] && h.stamp[k] == stamp) i = k;
  for (size_t k = 0; k < h.cap() && i == h.cap(); ++k) if (!h.used[k]) i = k;
  if (i == h.cap()) {
    for (size_t k = 0; k < h.cap(); ++k) if (oldest == h.cap() || h.stamp[k] < h.stamp[oldest]) oldest = k;
    if (stamp < h.stamp[oldest]) return ESVO_OK;
    i = oldest;
  }
  const size_t nimg = (size_t)c->dc.pitch * c->dc.H;
  // Both copies go on camera 0's time-surface stream behind both builds; camera 1's stream waits for them before it may
  // overwrite its image.  No host sync.
  cudaStream_t s0 = c->s_tsc[0], s1 = c->s_tsc[1];
  if (s1 != s0) { ESVO_CUDA_TRY(c, cudaEventRecord(h.ev_join, s1)); ESVO_CUDA_TRY(c, cudaStreamWaitEvent(s0, h.ev_join, 0)); }
  ESVO_CUDA_TRY(c, cudaStreamWaitEvent(s0, h.ev[i], 0));                  // a hand-over may still be reading the entry
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h.buf + 2 * i * nimg, c->ts[0].last_img, nimg, cudaMemcpyDeviceToDevice, s0));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(h.buf + (2 * i + 1) * nimg, c->ts[1].last_img, nimg, cudaMemcpyDeviceToDevice, s0));
  ESVO_CUDA_TRY(c, cudaEventRecord(h.ev[i], s0));
  if (s1 != s0) ESVO_CUDA_TRY(c, cudaStreamWaitEvent(s1, h.ev[i], 0));
  h.stamp[i] = stamp; h.used[i] = true;
  return ESVO_OK;
}
ESVO_API int esvo_set_ts_pair_stored_dev(esvo_ctx* c, int64_t stamp, const double T[16]) {
  CHECK_CTX(c);
  if (!T) return ESVO_ERR_INVALID_ARG;
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  Ctx::TsHistory& h = c->hist;
  size_t i = h.cap();
  for (size_t k = 0; k < h.cap(); ++k) if (h.used[k] && h.stamp[k] == stamp) { i = k; break; }
  if (i == h.cap()) {
    c->set_error("esvo_set_ts_pair_stored_dev: no time-surface pair is stored under stamp " + std::to_string((long long)stamp));
    return ESVO_ERR_STATE;
  }
  SlotBufs& f = c->slot();
  const size_t nimg = (size_t)c->dc.pitch * c->dc.H;
  ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->stream, h.ev[i], 0));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.obs_l, h.buf + 2 * i * nimg, nimg, cudaMemcpyDeviceToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.obs_r, h.buf + (2 * i + 1) * nimg, nimg, cudaMemcpyDeviceToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaEventRecord(h.ev[i], c->stream));
  return obs_set_pose(c, T);
}

ESVO_API int esvo_set_ts_pair_dev(esvo_ctx* c, const double T[16]) {
  CHECK_CTX(c);
  if (!T) return ESVO_ERR_INVALID_ARG;
  if (!c->ts[0].built || !c->ts[1].built) { c->set_error("esvo_set_ts_pair_dev needs a built time surface for both cameras"); return ESVO_ERR_STATE; }
  // begin a new frame: rotate to the next pipeline slot
  c->activate((int)(c->frame_no % (uint64_t)c->depth));
  SlotBufs& sl = c->slot();
  // Hand the two freshly built images to the slot WITHOUT copying: swap the slot's observation buffers with
  // the time-surface output buffers.  The buffers the TS state receives in exchange are overwritten by the
  // next build, so the TS stream must first wait until the slot's previous frame stopped reading them.
  if (c->s_tsc[1] != c->s_tsc[0]) {                              // join the right camera's stream into the left one
    ESVO_CUDA_TRY(c, cudaEventRecord(c->ev_ts_join, c->s_tsc[1]));
    ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->s_tsc[0], c->ev_ts_join, 0));
  }
  ESVO_CUDA_TRY(c, cudaEventRecord(sl.ev_obs, c->s_tsc[0]));    // both builds of this frame are complete at this point
  if (sl.ev_free_valid) {
    ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->s_tsc[0], sl.ev_free, 0));
    if (c->s_tsc[1] != c->s_tsc[0]) ESVO_CUDA_TRY(c, cudaStreamWaitEvent(c->s_tsc[1], sl.ev_free, 0));
  }
  for (int cam = 0; cam < 2; ++cam) {
    TsState& t = c->ts[cam];
    if (t.last_img != t.img_out) { c->set_error("esvo_set_ts_pair_dev: time surface not rebuilt since the last hand-off"); return ESVO_ERR_STATE; }
    uint8_t*& mine = cam == 0 ? sl.obs_l : sl.obs_r;
    std::swap(mine, t.img_out);
    t.last_img = mine;
  }
  if (!c->prm.smooth_time_surface) { sl.obs_ls = sl.obs_l; sl.obs_rs = sl.obs_r; }   // otherwise smooth_obs() fills obs_ls/obs_rs
  std::memcpy(sl.T_world_left, T, sizeof(sl.T_world_left));
  rigid_inverse(T, sl.T_left_world_inv);     // travels to the LM kernel by value: no upload, nothing pinned to guard
  c->obs_set = true;
  return ESVO_OK;
}

static int run_bm_stage(esvo_ctx* c) {
  if (c->prm.smooth_time_surface) { int rc = smooth_obs(c); if (rc) return rc; }  // EventBM.cpp:68-72
  ESVO_CUDA_TRY(c, cudaMemsetAsync(c->slot().d_counters, 0, kCounters * 8, c->stream));
  cudaEvent_t pe = c->prof_begin(1);
  int rc = bm_run(c);
  c->prof_end(pe);
  if (rc) return rc;
  return seeds_order(c);
}

ESVO_API int esvo_bm_match(esvo_ctx* c, const uint16_t* ex, const uint16_t* ey, const int64_t* et, size_t n,
                           const int64_t* pt, const double* poses, size_t np, esvo_seed* out, size_t* n_seeds,
                           uint64_t* n_evals) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  if (!c->obs_set) return ESVO_ERR_STATE;
  if (!n_seeds || (n && (!ex || !ey || !et))) return ESVO_ERR_INVALID_ARG;
  int rc = stage_inputs_packed(c, ex, ey, et, n, pt, poses, np);
  if (rc) return rc;
  if ((rc = run_bm_stage(c))) return rc;
  if ((rc = fetch_counters(c))) return rc;
  const SlotBufs& f = c->slot();
  const size_t cnt = (size_t)f.h_counters[1];
  if (n_evals) *n_evals = f.h_counters[5];
  if (cnt > *n_seeds) { *n_seeds = cnt; return ESVO_ERR_CAPACITY; }
  if (cnt) ESVO_CUDA_TRY(c, cudaMemcpy(out, f.d_seeds, cnt * sizeof(esvo_seed), cudaMemcpyDeviceToHost));
  *n_seeds = cnt;
  return ESVO_OK;
}


ESVO_API int esvo_depth_solve(esvo_ctx* c, const esvo_seed* seeds, size_t n, esvo_depth_point* out, size_t* n_out,
                              uint64_t* n_evals) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  if (!c->obs_set) return ESVO_ERR_STATE;
  if (!n_out || (n && !seeds)) return ESVO_ERR_INVALID_ARG;
  if (n == 0) { *n_out = 0; if (n_evals) *n_evals = 0; return ESVO_OK; }
  SlotBufs& f = c->slot();
  int rc = map_alloc_inputs(c, std::max(n, f.n_ev), f.n_poses);
  if (rc) return rc;
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(f.d_seeds, seeds, n * sizeof(esvo_seed), cudaMemcpyHostToDevice, c->stream));
  ESVO_CUDA_TRY(c, cudaMemsetAsync(f.d_counters, 0, kCounters * 8, c->stream));
  { cudaEvent_t pe = c->prof_begin(3); rc = lm_run(c, f.d_seeds, n); c->prof_end(pe); }
  if (rc) return rc;
  if ((rc = points_order_impl(c, f.d_seeds, n, 0, 0, 0, 0, 0, nullptr, nullptr))) return rc;
  if ((rc = fetch_counters(c))) return rc;
  const size_t cnt = (size_t)f.h_counters[3];
  if (n_evals) *n_evals = f.h_counters[6];
  if (cnt > *n_out) { *n_out = cnt; return ESVO_ERR_CAPACITY; }
  if (cnt) ESVO_CUDA_TRY(c, cudaMemcpy(out, f.d_pts, cnt * sizeof(esvo_depth_point), cudaMemcpyDeviceToHost));
  *n_out = cnt;
  return ESVO_OK;
}

}  // extern "C"
