// esvo_b200 product code -- camera tracking on the negative time surface (sm_90a).
//
// Replaces esvo_core::core::RegProblemLM::{setProblem, setStochasticSampling, operator(), thread,
// df, getWarpingTransformation, addMotionUpdate, setPose, reprojection, isValidPatch}
// (esvo_core/src/core/RegProblemLM.cpp:24-416), RegProblemSolverLM::{resetRegProblem,
// solve_analytical, solve_numerical} (esvo_core/src/core/RegProblemSolverLM.cpp:45-217),
// TimeSurfaceObservation::{getTimeSurfaceNegative, computeTsNegativeGrad}
// (esvo_core/include/esvo_core/container/TimeSurfaceObservation.h:118-147), tools::cayley2rot
// (esvo_core/src/tools/cayley.cpp:4-21) and the n = 6 instance of Eigen's LevenbergMarquardt
// (ColPivHouseholderQR + lmpar2 + qrsolv).
//
// Design: the whole solve (<= MAX_ITERATION outer iterations x {residual, analytic Jacobian,
// pivoted Householder QR of the B x 6 Jacobian, lmpar, trial residuals, compositional pose update})
// is ONE kernel launch of one thread block: the block is the batch (one thread per map point,
// B <= 1024), the Jacobian lives in shared memory, every norm / dot product is a block reduction
// and the 6x6 trust-region algebra runs on thread 0 between barriers.  The negative TS is kept as
// u8 (255 - blur is an exact integer) and its Sobel gradients as int16 (exact integers).
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace esvo {

constexpr int TRK_THREADS = 256;   // 8 warps: the scalar trust-region algebra on thread 0 gets up to 255 registers (no spills in the unrolled qrsolv)
constexpr int TRK_MAXB = 1024;

struct TrkDev {
  uint8_t* ts = nullptr;        // H*pitch current left TS
  uint8_t* neg = nullptr;       // H*pitch negative TS
  int16_t *du = nullptr, *dv = nullptr;  // H*W Sobel of the negative TS
  float* xyz = nullptr;         // permuted world points (numPoints*3)
  double* items = nullptr;      // ResItems: numPoints*3 in the ref frame
  double* state = nullptr;      // [0..8] R_, [9..11] t_, [12..27] T_world_ref, [28..43] T_world_left out, [44..46] stats
  size_t cap = 0;
  // device form (esvo_track_adopt_map_dev / esvo_track_reset_dev): snapshot of a published cloud and the uploaded sample indices
  float* ref = nullptr; size_t ref_cap = 0;
  int32_t* idx = nullptr; size_t idx_cap = 0;
};
struct TrackState {
  TrkDev d;
  size_t numPoints = 0, numBatches = 1;
  bool ready = false;
  // The adopted cloud stays where it is; ref->vPointXYZ_'s in-place shuffle becomes this index permutation of it, carried
  // from reset to reset like the reference's shuffled vector.
  std::vector<int32_t> perm;
  bool adopted = false;
  // glibc TYPE_3 rand() state (the reference calls the process-global rand(), RegProblemLM.cpp:49)
  uint32_t hist[31]; int pos = 0;
  void srand_(unsigned s) {
    if (s == 0) s = 1;
    std::vector<uint32_t> v(344);
    int32_t w = (int32_t)s; v[0] = (uint32_t)w;
    for (int i = 1; i < 31; ++i) { long hi = w / 127773, lo = w % 127773; w = (int32_t)(16807 * lo - 2836 * hi); if (w < 0) w += 2147483647; v[i] = (uint32_t)w; }
    for (int i = 31; i < 34; ++i) v[i] = v[i - 31];
    for (int i = 34; i < 344; ++i) v[i] = v[i - 31] + v[i - 3];
    for (int i = 0; i < 31; ++i) hist[i] = v[313 + i];
    pos = 0;
  }
  int rand_() { uint32_t n = hist[pos] + hist[(pos + 28) % 31]; hist[pos] = n; pos = (pos + 1) % 31; return (int)(n >> 1); }
};

// ---- negative TS: 255 - GaussianBlur5x5(u8) (kernelSize 5) or 255 - TS (kernelSize 0) ----
__device__ __forceinline__ int refl101t(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
  return p;
}
__global__ void trk_negative_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ neg, int W, int H, int pitch, int ksize) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  int v;
  if (ksize == 5) {
    const int k[5] = {1, 4, 6, 4, 1};
    int s = 0;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
      const uint8_t* row = src + (size_t)refl101t(y + dy, H) * pitch;
      int r = 0;
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx) r += k[dx + 2] * row[refl101t(x + dx, W)];
      s += k[dy + 2] * r;
    }
    v = (s + 128) >> 8;
  } else if (ksize == 3) {
    const int k[3] = {1, 2, 1};
    int s = 0;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      const uint8_t* row = src + (size_t)refl101t(y + dy, H) * pitch;
      int r = 0;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) r += k[dx + 1] * row[refl101t(x + dx, W)];
      s += k[dy + 1] * r;
    }
    v = (s + 8) >> 4;
  } else v = src[(size_t)y * pitch + x];
  neg[(size_t)y * pitch + x] = (uint8_t)(255 - v);
}
// cv::Sobel(CV_64F, ksize 3, BORDER_REFLECT_101), exact in integers
__global__ void trk_sobel_kernel(const uint8_t* __restrict__ neg, int16_t* __restrict__ du, int16_t* __restrict__ dv, int W, int H, int pitch) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const int xm = refl101t(x - 1, W), xp = refl101t(x + 1, W), ym = refl101t(y - 1, H), yp = refl101t(y + 1, H);
  auto S = [&](int xx, int yy) -> int { return neg[(size_t)yy * pitch + xx]; };
  du[(size_t)y * W + x] = (int16_t)((S(xp, ym) - S(xm, ym)) + 2 * (S(xp, y) - S(xm, y)) + (S(xp, yp) - S(xm, yp)));
  dv[(size_t)y * W + x] = (int16_t)((S(xm, yp) - S(xm, ym)) + 2 * (S(x, yp) - S(x, ym)) + (S(xp, yp) - S(xp, ym)));
}
// RegProblemLM::setProblem point transform (:53-54): p_cam = R_world_ref^T (p - t_world_ref)
// idx (device form): point i is xyz[idx[i]], the adopted cloud read through the sampling permutation
__global__ void trk_items_kernel(const float* __restrict__ xyz, const int32_t* __restrict__ idx, int n, const double* __restrict__ Twr,
                                 double* __restrict__ items) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t k = idx ? (size_t)idx[i] : (size_t)i;
  const double d0 = (double)xyz[3 * k] - Twr[3], d1 = (double)xyz[3 * k + 1] - Twr[7], d2 = (double)xyz[3 * k + 2] - Twr[11];
#pragma unroll
  for (int r = 0; r < 3; ++r) items[3 * i + r] = Twr[0 * 4 + r] * d0 + Twr[1 * 4 + r] * d1 + Twr[2 * 4 + r] * d2;
}

// ---------------------------------------------------------------------------------------------
// device-side 3x3 helpers
// ---------------------------------------------------------------------------------------------
__device__ void cayley2rot_d(const double* c, double* R) {
  const double scale = 1 + c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
  R[0] = 1 + c[0] * c[0] - c[1] * c[1] - c[2] * c[2]; R[1] = 2 * (c[0] * c[1] - c[2]); R[2] = 2 * (c[0] * c[2] + c[1]);
  R[3] = 2 * (c[0] * c[1] + c[2]); R[4] = 1 - c[0] * c[0] + c[1] * c[1] - c[2] * c[2]; R[5] = 2 * (c[1] * c[2] - c[0]);
  R[6] = 2 * (c[0] * c[2] - c[1]); R[7] = 2 * (c[1] * c[2] + c[0]); R[8] = 1 - c[0] * c[0] - c[1] * c[1] + c[2] * c[2];
  for (int i = 0; i < 9; ++i) R[i] = (1 / scale) * R[i];
}
__device__ void mul3_d(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
// U V^T of the SVD of M (JacobiSVD in the reference) = orthogonal polar factor M (M^T M)^{-1/2}
__device__ void polar_d(const double* M, double* Q) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i * 3 + j] = M[i] * M[j] + M[3 + i] * M[3 + j] + M[6 + i] * M[6 + j];
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = A[p * 3 + q];
        if (apq == 0) continue;
        const double theta = (A[q * 3 + q] - A[p * 3 + p]) / (2 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1));
        const double c = 1 / sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 3; ++k) { double a = A[k * 3 + p], b = A[k * 3 + q]; A[k * 3 + p] = c * a - s * b; A[k * 3 + q] = s * a + c * b; }
        for (int k = 0; k < 3; ++k) { double a = A[p * 3 + k], b = A[q * 3 + k]; A[p * 3 + k] = c * a - s * b; A[q * 3 + k] = s * a + c * b; }
        for (int k = 0; k < 3; ++k) { double a = V[k * 3 + p], b = V[k * 3 + q]; V[k * 3 + p] = c * a - s * b; V[k * 3 + q] = s * a + c * b; }
      }
  }
  const double isq[3] = {1 / sqrt(A[0]), 1 / sqrt(A[4]), 1 / sqrt(A[8])};
  double S[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) S[i * 3 + j] = V[i * 3] * isq[0] * V[j * 3] + V[i * 3 + 1] * isq[1] * V[j * 3 + 1] + V[i * 3 + 2] * isq[2] * V[j * 3 + 2];
  mul3_d(M, S, Q);
}
__device__ double det3_d(const double* A) {
  return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

// ---------------------------------------------------------------------------------------------
// n = 6 trust-region algebra on one thread (Eigen internal::qrsolv / lmpar2)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void givens_d(double p, double q, double& c, double& s) {
  // Eigen JacobiRotation::makeGivens (real).  The quotient and 1/sqrt(1+t^2) use the branch-free Newton forms of common.cuh
  // (<= 1 ulp; t in [-1,1] so 1+t^2 is in [1,2]) unless the divisor is outside the range they cover: on one thread of a block
  // that waits at a barrier, the latency of this chain (21 rotations per qrsolv, up to 10 qrsolv per lmpar) IS the solver's time.
  if (q == 0) { c = p < 0 ? -1 : 1; s = 0; }
  else if (p == 0) { c = 0; s = q < 0 ? 1 : -1; }
  else if (fabs(p) > fabs(q)) {
    if (fabs(p) > 1e-280 && fabs(p) < 1e280) { const double t = div_nr(q, p), r = rsqrt_nr(1 + t * t); c = p < 0 ? -r : r; s = -t * c; }
    else { double t = q / p, u = sqrt(1 + t * t); if (p < 0) u = -u; c = 1 / u; s = -t * c; }
  } else {
    if (fabs(q) > 1e-280 && fabs(q) < 1e280) { const double t = div_nr(p, q), r = rsqrt_nr(1 + t * t); s = q < 0 ? r : -r; c = -t * s; }
    else { double t = p / q, u = sqrt(1 + t * t); if (q < 0) u = -u; s = -1 / u; c = -t * s; }
  }
}
__device__ double norm6(const double* v) { double s = 0; for (int i = 0; i < 6; ++i) s += v[i] * v[i]; return sqrt(s); }

// s: 6x6 (row i, col j at s[j*6+i]); upper triangle = R.  dperm[j] = diag[ipvt[j]].  Every loop has compile-time bounds and is
// fully unrolled, so s / sdiag / wa live in registers (the rolled form kept them in local memory: an L1 round trip inside
// every step of the dependent rotation chain).
__device__ void qrsolv6(double* s, const int* ipvt, const double* dperm, const double* qtb, double* x, double* sdiag) {
  constexpr int n = 6;
  double wa[6];
#pragma unroll
  for (int j = 0; j < n; ++j) { x[j] = s[j * 6 + j]; wa[j] = qtb[j]; sdiag[j] = 0; }
#pragma unroll
  for (int j = 0; j < n; ++j)
#pragma unroll
    for (int i = j + 1; i < n; ++i) s[j * 6 + i] = s[i * 6 + j];
  bool live = true;
#pragma unroll
  for (int j = 0; j < n; ++j) {
    if (dperm[j] == 0.) live = false;        // MINPACK: "if (diag[l] == 0) break" out of the elimination loop
    if (live) {
#pragma unroll
      for (int k = j; k < n; ++k) sdiag[k] = 0;
      sdiag[j] = dperm[j];
      double qtbpj = 0.;
#pragma unroll
      for (int k = j; k < n; ++k) {
        double c, sn;
        givens_d(-s[k * 6 + k], sdiag[k], c, sn);
        s[k * 6 + k] = c * s[k * 6 + k] + sn * sdiag[k];
        double temp = c * wa[k] + sn * qtbpj;
        qtbpj = -sn * wa[k] + c * qtbpj;
        wa[k] = temp;
#pragma unroll
        for (int i = k + 1; i < n; ++i) {
          temp = c * s[k * 6 + i] + sn * sdiag[i];
          sdiag[i] = -sn * s[k * 6 + i] + c * sdiag[i];
          s[k * 6 + i] = temp;
        }
      }
    }
  }
  int nsing = n;
#pragma unroll
  for (int j = n - 1; j >= 0; --j) if (sdiag[j] == 0) nsing = j;      // first zero of sdiag
#pragma unroll
  for (int j = 0; j < n; ++j) if (j >= nsing) wa[j] = 0;
#pragma unroll
  for (int i = n - 1; i >= 0; --i) {
    if (i < nsing) {
      double sum = wa[i];
#pragma unroll
      for (int j = i + 1; j < n; ++j) if (j < nsing) sum -= s[i * 6 + j] * wa[j];
      wa[i] = sum / s[i * 6 + i];
    }
  }
#pragma unroll
  for (int j = 0; j < n; ++j) sdiag[j] = s[j * 6 + j];
#pragma unroll
  for (int j = 0; j < n; ++j) s[j * 6 + j] = x[j];
#pragma unroll
  for (int j = 0; j < n; ++j) x[ipvt[j]] = wa[j];
}

// R: 6x6 col-major upper; perm; rank
__device__ void lmpar6(const double* R, const int* perm, int rank, const double* diag, const double* qtb, double delta,
                       double& par, double* x) {
  const double dwarf = 2.2250738585072014e-308;
  const int n = 6;
  double wa1[6], wa2[6];
  for (int j = 0; j < n; ++j) wa1[j] = j < rank ? qtb[j] : 0;
  for (int i = rank - 1; i >= 0; --i) {
    double sum = wa1[i];
    for (int j = i + 1; j < rank; ++j) sum -= R[j * 6 + i] * wa1[j];
    wa1[i] = sum / R[i * 6 + i];
  }
  for (int j = 0; j < n; ++j) x[perm[j]] = wa1[j];
  int iter = 0;
  for (int j = 0; j < n; ++j) wa2[j] = diag[j] * x[j];
  double dxnorm = norm6(wa2);
  double fp = dxnorm - delta;
  if (fp <= 0.1 * delta) { par = 0; return; }
  double parl = 0.;
  if (rank == n) {
    for (int j = 0; j < n; ++j) wa1[j] = diag[perm[j]] * wa2[perm[j]] / dxnorm;
    for (int i = 0; i < n; ++i) {
      double sum = wa1[i];
      for (int j = 0; j < i; ++j) sum -= R[i * 6 + j] * wa1[j];
      wa1[i] = sum / R[i * 6 + i];
    }
    const double temp = norm6(wa1);
    parl = fp / delta / temp / temp;
  }
  for (int j = 0; j < n; ++j) {
    double sum = 0;
    for (int i = 0; i <= j; ++i) sum += R[j * 6 + i] * qtb[i];
    wa1[j] = sum / diag[perm[j]];
  }
  const double gnorm = norm6(wa1);
  double paru = gnorm / delta;
  if (paru == 0.) paru = dwarf / fmin(delta, 0.1);
  par = fmax(par, parl);
  par = fmin(par, paru);
  if (par == 0.) par = gnorm / dxnorm;
  double s[36], sdiag[6];
  for (int i = 0; i < 36; ++i) s[i] = R[i];
  while (true) {
    ++iter;
    if (par == 0.) par = fmax(dwarf, .001 * paru);
    const double sp = sqrt(par);
    for (int j = 0; j < n; ++j) wa1[j] = sp * diag[perm[j]];      // qrsolv's diag[ipvt[j]], gathered once
    qrsolv6(s, perm, wa1, qtb, x, sdiag);
    for (int j = 0; j < n; ++j) wa2[j] = diag[j] * x[j];
    dxnorm = norm6(wa2);
    double temp = fp;
    fp = dxnorm - delta;
    if (fabs(fp) <= 0.1 * delta || (parl == 0. && fp <= temp && temp < 0.) || iter == 10) break;
    for (int j = 0; j < n; ++j) wa1[j] = diag[perm[j]] * (wa2[perm[j]] / dxnorm);
    for (int j = 0; j < n; ++j) {
      wa1[j] /= sdiag[j];
      temp = wa1[j];
      for (int i = j + 1; i < n; ++i) wa1[i] -= s[j * 6 + i] * temp;
    }
    temp = norm6(wa1);
    const double parc = fp / delta / temp / temp;
    if (fp > 0.) parl = fmax(parl, par);
    if (fp < 0.) paru = fmin(paru, par);
    par = fmax(parl, par + parc);
  }
  if (iter == 0) par = 0.;
}

// ---------------------------------------------------------------------------------------------
// block reductions (TRK_THREADS threads): sums of up to 6 values at once
// ---------------------------------------------------------------------------------------------
template <int K>
__device__ void block_sumK(double* v, double* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) s_red[warp * 8 + k] = v[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double t = 0;
    for (int w = 0; w < nw; ++w) t += s_red[w * 8 + k];   // same order in every thread -> identical bits
    v[k] = t;
  }
}

struct TrkArgs {
  const uint8_t* neg; const int16_t* du; const int16_t* dv; const uint8_t* mask;
  const double* items; int total; int numBatches; int batch; int max_iter; int huber; double huber_thr;
  int analytical; double* state;
};

__device__ __forceinline__ bool trk_reproject(const DevConsts& dc, const uint8_t* mask, const double* p, const double* T, double& x, double& y) {
  double pl[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) pl[r] = T[r * 4] * p[0] + T[r * 4 + 1] * p[1] + T[r * 4 + 2] * p[2] + T[r * 4 + 3];
  double h[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) h[r] = dc.Pl[r * 4] * pl[0] + dc.Pl[r * 4 + 1] * pl[1] + dc.Pl[r * 4 + 2] * pl[2] + dc.Pl[r * 4 + 3];
  x = h[0] / h[2]; y = h[1] / h[2];
  if (!(x == x) || !(y == y)) return false;
  if (x < 0 || x > dc.W - 1 || y < 0 || y > dc.H - 1) return false;              // isValidPatch, 1x1 (:380-400)
  if (mask[(size_t)((int)y) * dc.W + (int)x] < 125) return false;
  return true;
}
// patchInterpolation for a 1x1 patch (RegProblemLM.cpp:418-487)
template <class PixT>
__device__ __forceinline__ bool trk_interp(const DevConsts& dc, const PixT* img, int stride, double x, double y, double& out) {
  const int fx = (int)floor(x), fy = (int)floor(y);
  if (fx < 0 || fy < 0 || fx >= dc.W || fy >= dc.H) return false;
  if (fy + 1 >= dc.H || fx + 1 >= dc.W) return false;
  const double q1 = (fx + 1) - x, q2 = x - fx, q3 = (fy + 1) - y, q4 = y - fy;
  const PixT* a = img + (size_t)fy * stride + fx;
  const double a00 = (double)a[0], a01 = (double)a[1], a10 = (double)a[stride], a11 = (double)a[stride + 1];
  out = q3 * (q1 * a00 + q2 * a01) + q4 * (q1 * a10 + q2 * a11);
  return true;
}

__global__ void __launch_bounds__(TRK_THREADS) trk_solve_kernel(DevConsts dc, TrkArgs a) {
  extern __shared__ double smem[];
  double* sJ = smem;                          // TRK_MAXB x 6, column-major with leading dim mB
  double* sF = sJ + TRK_MAXB * 6;             // fvec (accepted)
  double* sF2 = sF + TRK_MAXB;                // trial fvec / wa4
  double* sP = sF2 + TRK_MAXB;                // batch points (3 per point)
  double* s_red = sP + TRK_MAXB * 3;          // 16 warps x 8
  __shared__ double sT[12], sR[9], st[3], sx[6], sTau[6], sNormU[6], sNormD[6], sScal[8];
  __shared__ int sPerm[6], sTransp[6], sCtl[4];
  const int tid = threadIdx.x;
  if (tid < 9) sR[tid] = a.state[tid];
  if (tid < 3) st[tid] = a.state[9 + tid];
  __syncthreads();
  const double EPS = 2.220446049250313e-16;
  const double ftol = 1e-3, xtol = 1e-3, factor = 100.;
  const int maxfev = a.max_iter * 8;
  long long nfev_total = 0;
  int iteration = 0, m = 0;

  // residual evaluation of the current batch at increment x6 (operator(), :91-136) -> out[], returns ||out||^2
  auto eval_residual = [&](const double* x6, double* out) -> double {
    if (tid == 0) {  // getWarpingTransformation (:322-346)
      double dR[9], dRt[9], Rt[9], newR[9], Rcr[9];
      cayley2rot_d(x6, dR);
      for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { dRt[i * 3 + j] = dR[j * 3 + i]; Rt[i * 3 + j] = sR[j * 3 + i]; }
      mul3_d(Rt, dRt, newR);
      polar_d(newR, Rcr);
      sCtl[3] = det3_d(Rcr) < 0.0 ? 1 : 0;
      double v[3];
      for (int i = 0; i < 3; ++i) v[i] = x6[3 + i] + dR[i * 3] * st[0] + dR[i * 3 + 1] * st[1] + dR[i * 3 + 2] * st[2];
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) sT[i * 4 + j] = Rcr[i * 3 + j];
        sT[i * 4 + 3] = -(Rcr[i * 3] * v[0] + Rcr[i * 3 + 1] * v[1] + Rcr[i * 3 + 2] * v[2]);
      }
    }
    __syncthreads();
    double ss[1] = {0};
    for (int i = tid; i < m; i += blockDim.x) {
      double x, y, r = 255.0, tau;
      if (trk_reproject(dc, a.mask, &sP[3 * i], sT, x, y) && trk_interp<uint8_t>(dc, a.neg, dc.pitch, x, y, tau)) r = tau;
      if (a.huber) { double w = 1.0; if (r > a.huber_thr) w = a.huber_thr / r; r = sqrt(w) * r; }
      out[i] = r;
      ss[0] += r * r;
    }
    block_sumK<1>(ss, s_red);
    return ss[0];
  };

  while (true) {
    if (iteration >= a.max_iter) break;
    // ---- setStochasticSampling (:70-89) ----
    const int offset = (iteration % a.numBatches) * a.batch;
    m = min(a.batch, a.total - offset);
    if (m < 0) m = 0;
    __syncthreads();
    for (int i = tid; i < 3 * m; i += blockDim.x) sP[i] = a.items[3 * offset + i];
    if (tid < 6) sx[tid] = 0.0;
    __syncthreads();
    if (m < 6) break;  // minimizeInit: ImproperInputParameters (m < n)
    // ---- minimizeInit ----
    int nfev = 1;
    double fnorm = sqrt(eval_residual(sx, sF));
    double par = 0.; int iter = 1;
    // ---- minimizeOneStep ----
    int status = -1;
    // Jacobian
    if (a.analytical) {  // df (:178-269) at x = 0
      __shared__ double sJc[6], sTl[12];
      if (tid == 0) {
        for (int i = 0; i < 3; ++i) { sJc[i * 2] = sR[0 * 3 + i] * (1.0 / dc.Pl[0]); sJc[i * 2 + 1] = sR[1 * 3 + i] * (1.0 / dc.Pl[5]); }
        for (int i = 0; i < 3; ++i) {
          for (int j = 0; j < 3; ++j) sTl[i * 4 + j] = sR[j * 3 + i];
          sTl[i * 4 + 3] = -(sR[0 * 3 + i] * st[0] + sR[1 * 3 + i] * st[1] + sR[2 * 3 + i] * st[2]);
        }
      }
      __syncthreads();
      for (int i = tid; i < m; i += blockDim.x) {
        const double* p = &sP[3 * i];
        double row12[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) row12[k] = 0;
        double x, y, gx, gy;
        if (trk_reproject(dc, a.mask, p, sTl, x, y) && trk_interp<int16_t>(dc, a.du, dc.W, x, y, gx) &&
            trk_interp<int16_t>(dc, a.dv, dc.W, x, y, gy)) {
          const double g0 = gx / 8, g1 = gy / 8;
          double dPi[6] = {dc.Pl[0] / p[2], dc.Pl[1] / p[2], 0, dc.Pl[4] / p[2], dc.Pl[5] / p[2], 0};
          const double z2 = p[2] * p[2];
          dPi[2] = -(dc.Pl[0] * p[0] + dc.Pl[1] * p[1] + dc.Pl[3]) / z2;
          dPi[5] = -(dc.Pl[4] * p[0] + dc.Pl[5] * p[1] + dc.Pl[7]) / z2;
          double aa[3], bb[2], cc[3];
          for (int k = 0; k < 3; ++k) aa[k] = g0 * dPi[k] + g1 * dPi[3 + k];
          for (int k = 0; k < 2; ++k) bb[k] = aa[0] * sJc[k] + aa[1] * sJc[2 + k] + aa[2] * sJc[4 + k];
          for (int k = 0; k < 3; ++k) cc[k] = bb[0] * dPi[k] + bb[1] * dPi[3 + k];
          for (int blk = 0; blk < 4; ++blk) {
            const double s = blk < 3 ? p[blk] : 1.0;
            for (int k = 0; k < 3; ++k) row12[blk * 3 + k] = (cc[k] * s) * p[2];
          }
        }
        // fjac = -fjacBlock * J_G_0 (J_G_0: A1=[[0,0,0],[0,0,2],[0,-2,0]], A2=[[0,0,-2],[0,0,0],[2,0,0]], A3=[[0,2,0],[-2,0,0],[0,0,0]], I)
        sJ[0 * m + i] = -(2 * row12[5] + -2 * row12[7]);
        sJ[1 * m + i] = -(-2 * row12[2] + 2 * row12[6]);
        sJ[2 * m + i] = -(2 * row12[1] + -2 * row12[3]);
        sJ[3 * m + i] = -row12[9];
        sJ[4 * m + i] = -row12[10];
        sJ[5 * m + i] = -row12[11];
      }
      __syncthreads();
    } else {  // NumericalDiff<Forward> (n+1 = 7 evaluations, the first repeats f(0))
      const double h = 1.4901161193847656e-08;
      for (int j = 0; j < 6; ++j) {
        __shared__ double sxh[6];
        if (tid < 6) sxh[tid] = (tid == j) ? h : 0.0;
        __syncthreads();
        eval_residual(sxh, sF2);
        for (int i = tid; i < m; i += blockDim.x) sJ[j * m + i] = (sF2[i] - sF[i]) / h;
        __syncthreads();
      }
      nfev += 7;
    }
    // wa2 = column norms
    double wa2[6];
    {
      double cs[6] = {0, 0, 0, 0, 0, 0};
      for (int i = tid; i < m; i += blockDim.x)
#pragma unroll
        for (int j = 0; j < 6; ++j) cs[j] += sJ[j * m + i] * sJ[j * m + i];
      block_sumK<6>(cs, s_red);
#pragma unroll
      for (int j = 0; j < 6; ++j) wa2[j] = sqrt(cs[j]);
    }
    // ---- ColPivHouseholderQR (Eigen 3.3 computeInPlace) in place on sJ ----
    if (tid < 6) { sNormU[tid] = wa2[tid]; sNormD[tid] = wa2[tid]; }
    __syncthreads();
    double maxpivot = 0; int nonzero_pivots = 6;
    {
      double mx = 0;
      for (int j = 0; j < 6; ++j) mx = fmax(mx, wa2[j]);
      const double th = (mx * EPS / m) * (mx * EPS / m);
      const double downdate_thr = sqrt(EPS);
      for (int k = 0; k < 6; ++k) {
        int big = k; double bigv = sNormU[k];
        for (int j = k + 1; j < 6; ++j) if (sNormU[j] > bigv) { bigv = sNormU[j]; big = j; }
        if (nonzero_pivots == 6 && bigv * bigv < th * (double)(m - k)) nonzero_pivots = k;
        __syncthreads();
        if (tid == 0) {
          sTransp[k] = big;
          if (k != big) { double t = sNormU[k]; sNormU[k] = sNormU[big]; sNormU[big] = t; t = sNormD[k]; sNormD[k] = sNormD[big]; sNormD[big] = t; }
        }
        if (k != big) for (int i = tid; i < m; i += blockDim.x) { double t = sJ[k * m + i]; sJ[k * m + i] = sJ[big * m + i]; sJ[big * m + i] = t; }
        __syncthreads();
        const double c0 = sJ[k * m + k];
        double ts[1] = {0};
        for (int i = tid; i < m; i += blockDim.x) if (i > k) ts[0] += sJ[k * m + i] * sJ[k * m + i];
        block_sumK<1>(ts, s_red);
        double beta, tau;
        if (ts[0] <= 2.2250738585072014e-308) { tau = 0; beta = c0; for (int i = tid; i < m; i += blockDim.x) if (i > k) sJ[k * m + i] = 0; }
        else {
          beta = sqrt(c0 * c0 + ts[0]);
          if (c0 >= 0) beta = -beta;
          for (int i = tid; i < m; i += blockDim.x) if (i > k) sJ[k * m + i] = sJ[k * m + i] / (c0 - beta);
          tau = (beta - c0) / beta;
        }
        __syncthreads();
        if (tid == 0) { sTau[k] = tau; sJ[k * m + k] = beta; }
        if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
        // apply H_k to the trailing columns
        if (k < 5 && tau != 0) {
          double tm[6] = {0, 0, 0, 0, 0, 0};
          for (int i = tid; i < m; i += blockDim.x) if (i > k)
            for (int j = k + 1; j < 6; ++j) tm[j] += sJ[k * m + i] * sJ[j * m + i];
          block_sumK<6>(tm, s_red);
          for (int j = k + 1; j < 6; ++j) tm[j] += sJ[j * m + k];
          __syncthreads();
          for (int i = tid; i < m; i += blockDim.x) if (i > k)
            for (int j = k + 1; j < 6; ++j) sJ[j * m + i] -= tau * sJ[k * m + i] * tm[j];
          if (tid == 0) for (int j = k + 1; j < 6; ++j) sJ[j * m + k] -= tau * tm[j];
        }
        __syncthreads();
        // norm downdate
        for (int j = k + 1; j < 6; ++j) {
          const double nu_ = sNormU[j];
          if (nu_ != 0) {
            double temp = fabs(sJ[j * m + k]) / nu_;
            temp = (1 + temp) * (1 - temp);
            temp = temp < 0 ? 0 : temp;
            const double rr = nu_ / sNormD[j];
            const double temp2 = temp * rr * rr;
            if (temp2 <= downdate_thr) {
              double ds[1] = {0};
              for (int i = tid; i < m; i += blockDim.x) if (i > k) ds[0] += sJ[j * m + i] * sJ[j * m + i];
              block_sumK<1>(ds, s_red);
              __syncthreads();
              if (tid == 0) { sNormD[j] = sqrt(ds[0]); sNormU[j] = sNormD[j]; }
            } else {
              __syncthreads();
              if (tid == 0) sNormU[j] = nu_ * sqrt(temp);
            }
            __syncthreads();
          }
        }
      }
      if (tid == 0) {
        for (int j = 0; j < 6; ++j) sPerm[j] = j;
        for (int k = 0; k < 6; ++k) { int t = sPerm[k]; sPerm[k] = sPerm[sTransp[k]]; sPerm[sTransp[k]] = t; }
      }
      __syncthreads();
    }
    // qtf = first 6 entries of Q^T fvec
    for (int i = tid; i < m; i += blockDim.x) sF2[i] = sF[i];
    __syncthreads();
    for (int k = 0; k < 6; ++k) {
      const double tau = sTau[k];
      if (tau == 0) continue;
      double ds[1] = {0};
      for (int i = tid; i < m; i += blockDim.x) if (i > k) ds[0] += sJ[k * m + i] * sF2[i];
      block_sumK<1>(ds, s_red);
      const double tmp = ds[0] + sF2[k];
      __syncthreads();
      for (int i = tid; i < m; i += blockDim.x) if (i > k) sF2[i] -= tau * sJ[k * m + i] * tmp;
      if (tid == 0) sF2[k] -= tau * tmp;
      __syncthreads();
    }
    // ---- the rest of minimizeOneStep: scalar control on every thread (identical values), heavy 6x6 work on thread 0 ----
    double R[36], qtf[6], diag[6];
    int perm[6];
    for (int j = 0; j < 6; ++j) { perm[j] = sPerm[j]; qtf[j] = sF2[j]; for (int i = 0; i < 6; ++i) R[j * 6 + i] = (i <= j) ? sJ[j * m + i] : 0.0; }
    int rank = 0;
    { const double thr = fabs(maxpivot) * EPS * 6; for (int i = 0; i < nonzero_pivots; ++i) rank += (fabs(R[i * 6 + i]) > thr); }
    double xnorm, delta;
    for (int j = 0; j < 6; ++j) diag[j] = (wa2[j] == 0.) ? 1. : wa2[j];   // iter == 1 always (fresh minimizeInit)
    xnorm = 0;                                                             // x = 0
    delta = factor * xnorm;
    if (delta == 0.) delta = factor;
    double gnorm = 0.;
    if (fnorm != 0.)
      for (int j = 0; j < 6; ++j)
        if (wa2[perm[j]] != 0.) {
          double s = 0;
          for (int i = 0; i <= j; ++i) s += R[j * 6 + i] * (qtf[i] / fnorm);
          gnorm = fmax(gnorm, fabs(s / wa2[perm[j]]));
        }
    double xcur[6] = {0, 0, 0, 0, 0, 0};
    if (gnorm <= 0.) status = 4;
    else {
      for (int j = 0; j < 6; ++j) diag[j] = fmax(diag[j], wa2[j]);
      double ratio;
      do {
        __syncthreads();
        if (tid == 0) {
          double p6[6], parl = par;
          lmpar6(R, perm, rank, diag, qtf, delta, parl, p6);
          sScal[0] = parl;
          for (int j = 0; j < 6; ++j) sx[j] = -p6[j];
        }
        __syncthreads();
        par = sScal[0];
        double wa1[6], xn[6];
        for (int j = 0; j < 6; ++j) { wa1[j] = sx[j]; xn[j] = xcur[j] + wa1[j]; }
        double s = 0;
        for (int j = 0; j < 6; ++j) s += (diag[j] * wa1[j]) * (diag[j] * wa1[j]);
        const double pnorm = sqrt(s);
        if (iter == 1) delta = fmin(delta, pnorm);
        __syncthreads();
        if (tid < 6) sx[tid] = xn[tid];
        __syncthreads();
        const double fnorm1 = sqrt(eval_residual(sx, sF2));
        ++nfev;
        double actred = -1.;
        if (.1 * fnorm1 < fnorm) actred = 1. - (fnorm1 / fnorm) * (fnorm1 / fnorm);
        double wa3[6];
        for (int i = 0; i < 6; ++i) { double t = 0; for (int j = i; j < 6; ++j) t += R[j * 6 + i] * wa1[perm[j]]; wa3[i] = t; }
        const double t1 = norm6(wa3) / fnorm, temp1 = t1 * t1;
        const double t2 = sqrt(par) * pnorm / fnorm, temp2 = t2 * t2;
        const double prered = temp1 + temp2 / .5, dirder = -(temp1 + temp2);
        ratio = 0.;
        if (prered != 0.) ratio = actred / prered;
        if (ratio <= .25) {
          double temp = 0;
          if (actred >= 0.) temp = .5;
          if (actred < 0.) temp = .5 * dirder / (dirder + .5 * actred);
          if (.1 * fnorm1 >= fnorm || temp < .1) temp = .1;
          delta = temp * fmin(delta, pnorm / .1);
          par /= temp;
        } else if (!(par != 0. && ratio < .75)) { delta = pnorm / .5; par = .5 * par; }
        if (ratio >= 1e-4) {
          for (int j = 0; j < 6; ++j) xcur[j] = xn[j];
          double s2 = 0;
          for (int j = 0; j < 6; ++j) s2 += (diag[j] * xcur[j]) * (diag[j] * xcur[j]);
          xnorm = sqrt(s2);
          __syncthreads();
          for (int i = tid; i < m; i += blockDim.x) sF[i] = sF2[i];
          fnorm = fnorm1;
          ++iter;
        }
        if (fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1. && delta <= xtol * xnorm) { status = 3; break; }
        if (fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1.) { status = 1; break; }
        if (delta <= xtol * xnorm) { status = 2; break; }
        if (nfev >= maxfev) { status = 5; break; }
        if (fabs(actred) <= EPS && prered <= EPS && .5 * ratio <= 1.) { status = 6; break; }
        if (delta <= EPS * xnorm) { status = 7; break; }
        if (gnorm <= EPS) { status = 8; break; }
      } while (ratio < 1e-4);
    }
    // ---- addMotionUpdate (:348-360) ----
    __syncthreads();
    if (tid == 0) {
      double dR[9], newR[9], Rn[9], tn[3];
      cayley2rot_d(xcur, dR);
      mul3_d(dR, sR, newR);
      polar_d(newR, Rn);
      for (int i = 0; i < 3; ++i) tn[i] = xcur[3 + i] + dR[i * 3] * st[0] + dR[i * 3 + 1] * st[1] + dR[i * 3 + 2] * st[2];
      for (int i = 0; i < 9; ++i) sR[i] = Rn[i];
      for (int i = 0; i < 3; ++i) st[i] = tn[i];
    }
    __syncthreads();
    iteration++;
    nfev_total += nfev;
    if (status == 2 || status == 3) break;
  }
  // ---- setPose (:362-372) + statistics ----
  __syncthreads();
  if (tid == 0) {
    const double* Twr = a.state + 12;
    double* Tout = a.state + 28;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) Tout[i * 4 + j] = Twr[i * 4] * sR[j] + Twr[i * 4 + 1] * sR[3 + j] + Twr[i * 4 + 2] * sR[6 + j];
      Tout[i * 4 + 3] = Twr[i * 4] * st[0] + Twr[i * 4 + 1] * st[1] + Twr[i * 4 + 2] * st[2] + Twr[i * 4 + 3];
    }
    Tout[12] = 0; Tout[13] = 0; Tout[14] = 0; Tout[15] = 1;
    for (int i = 0; i < 9; ++i) a.state[i] = sR[i];
    for (int i = 0; i < 3; ++i) a.state[9 + i] = st[i];
    a.state[44] = (double)m; a.state[45] = (double)nfev_total; a.state[46] = (double)iteration;
  }
}

// ---------------------------------------------------------------------------------------------
int track_alloc(Ctx* c) {
  TrackState* t = new TrackState();
  c->trk = t;
  t->srand_(1);
  const size_t npix = (size_t)c->dc.W * c->dc.H, nimg = (size_t)c->dc.pitch * c->dc.H;
  TrkDev& d = t->d;
  ESVO_CUDA_TRY(c, dmalloc(&d.ts, nimg)); ESVO_CUDA_TRY(c, dmalloc(&d.neg, nimg));
  ESVO_CUDA_TRY(c, dmalloc(&d.du, npix)); ESVO_CUDA_TRY(c, dmalloc(&d.dv, npix));
  ESVO_CUDA_TRY(c, dmalloc(&d.state, 64));
  ESVO_CUDA_TRY(c, cudaMemset(d.ts, 0, nimg));
  d.cap = 4096;
  ESVO_CUDA_TRY(c, dmalloc(&d.xyz, d.cap * 3)); ESVO_CUDA_TRY(c, dmalloc(&d.items, d.cap * 3));
  static bool attr_set = false;
  (void)attr_set;
  const int smem = (TRK_MAXB * 6 + TRK_MAXB * 2 + TRK_MAXB * 3 + 16 * 8) * 8;
  ESVO_CUDA_TRY(c, cudaFuncSetAttribute(trk_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  return ESVO_OK;
}
void track_free(Ctx* c) {
  TrackState* t = c->trk;
  if (!t) return;
  void* ps[] = {t->d.ts, t->d.neg, t->d.du, t->d.dv, t->d.xyz, t->d.items, t->d.state, t->d.ref, t->d.idx};
  for (void* p : ps) if (p) cudaFree(p);
  delete t;
  c->trk = nullptr;
}

static bool inverse4_host(const double* A, double* inv) {
  double a[4][8];
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { a[i][j] = A[i * 4 + j]; a[i][4 + j] = (i == j); }
  for (int col = 0; col < 4; ++col) {
    int piv = col;
    for (int r = col + 1; r < 4; ++r) if (std::fabs(a[r][col]) > std::fabs(a[piv][col])) piv = r;
    if (a[piv][col] == 0) return false;
    if (piv != col) for (int j = 0; j < 8; ++j) std::swap(a[piv][j], a[col][j]);
    const double d = a[col][col];
    for (int j = 0; j < 8; ++j) a[col][j] /= d;
    for (int r = 0; r < 4; ++r) if (r != col) { const double f = a[r][col]; if (f != 0) for (int j = 0; j < 8; ++j) a[r][j] -= f * a[col][j]; }
  }
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) inv[i * 4 + j] = a[i][4 + j];
  return true;
}

// resetRegProblem / setProblem for both forms: ref_xyz != NULL is the caller's host cloud of n points, shuffled in place;
// ref_xyz == NULL is the adopted device cloud, shuffled through TrackState::perm.  Same rand() draws in the same order.
static int track_reset(esvo_ctx* c, float* ref_xyz, size_t n, const double Twr[16], const double Twc[16], const uint8_t* ts_left) {
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  const esvo_params& p = c->prm;
  if (p.trk_patch_size_x != 1 || p.trk_patch_size_y != 1) { c->set_error("tracking patch must be 1x1 (as in every shipped cfg)"); return ESVO_ERR_UNSUPPORTED; }
  if (p.trk_batch_size > TRK_MAXB || p.trk_batch_size < 6) { c->set_error("BATCH_SIZE must be in [6,1024]"); return ESVO_ERR_UNSUPPORTED; }
  if (p.trk_kernel_size != 0 && p.trk_kernel_size != 3 && p.trk_kernel_size != 5) { c->set_error("kernelSize must be 0, 3 or 5"); return ESVO_ERR_UNSUPPORTED; }
  if (n < (size_t)p.trk_batch_size) return 1;   // resetRegProblem: not enough points (RegProblemSolverLM.cpp:52-57)
  TrackState* t = c->trk;
  TrkDev& d = t->d;
  const DevConsts& dc = c->dc;
  // current TS
  if (ts_left) ESVO_CUDA_TRY(c, cudaMemcpy2DAsync(d.ts, dc.pitch, ts_left, dc.W, dc.W, dc.H, cudaMemcpyHostToDevice, c->stream));
  else {
    if (!c->ts[0].built) { c->set_error("ts_left == NULL but no time surface was built for camera 0"); return ESVO_ERR_STATE; }
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(d.ts, c->ts[0].last_img, (size_t)dc.pitch * dc.H, cudaMemcpyDeviceToDevice, c->stream));
  }
  // setProblem (:24-68): R_, t_ from T_ref_left = T_world_ref^-1 * T_world_left
  double inv[16], Trl[16];
  if (!inverse4_host(Twr, inv)) return ESVO_ERR_INVALID_ARG;
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += inv[i * 4 + k] * Twc[k * 4 + j]; Trl[i * 4 + j] = s; }
  double state[64] = {0};
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) state[i * 3 + j] = Trl[i * 4 + j]; state[9 + i] = Trl[i * 4 + 3]; }
  std::memcpy(state + 12, Twr, 128);
  std::memcpy(state + 28, Twc, 128);
  // stochastic sampling: partial Fisher-Yates driven by rand() (:45-50), in place on the cloud
  const size_t numPoints = std::min(n, (size_t)p.trk_max_registration_points);
  for (size_t i = 0; i < numPoints; ++i) {
    const size_t j = i + (size_t)t->rand_() % (n - i);
    if (ref_xyz) for (int k = 0; k < 3; ++k) std::swap(ref_xyz[3 * i + k], ref_xyz[3 * j + k]);
    else std::swap(t->perm[i], t->perm[j]);
  }
  if (numPoints > d.cap) {
    cudaFree(d.xyz); cudaFree(d.items);
    d.cap = numPoints;
    ESVO_CUDA_TRY(c, dmalloc(&d.xyz, d.cap * 3)); ESVO_CUDA_TRY(c, dmalloc(&d.items, d.cap * 3));
  }
  if (ref_xyz) ESVO_CUDA_TRY(c, cudaMemcpyAsync(d.xyz, ref_xyz, numPoints * 3 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  else {   // only the sampled indices travel; the cloud itself is never moved
    if (numPoints > d.idx_cap) { cudaFree(d.idx); d.idx_cap = numPoints; ESVO_CUDA_TRY(c, dmalloc(&d.idx, d.idx_cap)); }
    ESVO_CUDA_TRY(c, cudaMemcpyAsync(d.idx, t->perm.data(), numPoints * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  }
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(d.state, state, sizeof(state), cudaMemcpyHostToDevice, c->stream));
  trk_items_kernel<<<div_up((int)numPoints, 256), 256, 0, c->stream>>>(ref_xyz ? d.xyz : d.ref, ref_xyz ? nullptr : d.idx, (int)numPoints,
                                                                       d.state + 12, d.items);
  dim3 b(32, 8), g(div_up(dc.W, 32), div_up(dc.H, 8));
  trk_negative_kernel<<<g, b, 0, c->stream>>>(d.ts, d.neg, dc.W, dc.H, dc.pitch, p.trk_kernel_size);
  trk_sobel_kernel<<<g, b, 0, c->stream>>>(d.neg, d.du, d.dv, dc.W, dc.H, dc.pitch);
  c->launches += 3;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));   // state[] and perm live on the host
  t->numPoints = numPoints;
  t->numBatches = std::max(numPoints / (size_t)p.trk_batch_size, (size_t)1);
  t->ready = true;
  return ESVO_OK;
}

}  // namespace esvo

using namespace esvo;

extern "C" {

ESVO_API int esvo_track_srand(esvo_ctx* c, unsigned seed) { CHECK_CTX(c); c->trk->srand_(seed); return ESVO_OK; }

ESVO_API int esvo_track_reset(esvo_ctx* c, float* ref_xyz, size_t n, const double Twr[16], const double Twc[16],
                              const uint8_t* ts_left) {
  CHECK_CTX(c);
  if (!ref_xyz || !Twr || !Twc) return ESVO_ERR_INVALID_ARG;
  return track_reset(c, ref_xyz, n, Twr, Twc, ts_left);
}

ESVO_API int esvo_track_adopt_map_dev(esvo_ctx* c, int64_t stamp, size_t* n_points) {
  CHECK_CTX(c);
  if (int rc0 = drain_if_pipelined(c)) return rc0;
  const Ctx::Published& pb = c->pub;
  if (!pb.valid || pb.stamp != stamp) {
    c->set_error("esvo_track_adopt_map_dev: the newest cloud published on this context is not the one of stamp " + std::to_string((long long)stamp));
    return ESVO_ERR_STATE;
  }
  TrackState* t = c->trk;
  TrkDev& d = t->d;
  if (pb.n > d.ref_cap) { cudaFree(d.ref); d.ref_cap = pb.n; ESVO_CUDA_TRY(c, dmalloc(&d.ref, 3 * d.ref_cap)); }
  // a snapshot: the mapper may publish again before the next tracking pass
  if (pb.n) ESVO_CUDA_TRY(c, cudaMemcpyAsync(d.ref, pb.xyz, pb.n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  t->perm.resize(pb.n);
  for (size_t i = 0; i < pb.n; ++i) t->perm[i] = (int32_t)i;
  t->adopted = true;
  if (n_points) *n_points = pb.n;
  return ESVO_OK;
}

ESVO_API int esvo_track_reset_dev(esvo_ctx* c, const double Twr[16], const double Twc[16], const uint8_t* ts_left) {
  CHECK_CTX(c);
  if (!Twr || !Twc) return ESVO_ERR_INVALID_ARG;
  if (!c->trk->adopted) { c->set_error("esvo_track_reset_dev: no map adopted (esvo_track_adopt_map_dev)"); return ESVO_ERR_STATE; }
  return track_reset(c, nullptr, c->trk->perm.size(), Twr, Twc, ts_left);
}

ESVO_API int esvo_track_solve(esvo_ctx* c, int analytical, double Tout[16], esvo_lm_stats* st) {
  CHECK_CTX(c);
  TrackState* t = c->trk;
  if (!t->ready) return ESVO_ERR_STATE;
  if (!Tout) return ESVO_ERR_INVALID_ARG;
  const esvo_params& p = c->prm;
  TrkArgs a;
  a.neg = t->d.neg; a.du = t->d.du; a.dv = t->d.dv; a.mask = c->d_mask; a.items = t->d.items; a.total = (int)t->numPoints;
  a.numBatches = (int)t->numBatches; a.batch = p.trk_batch_size; a.max_iter = p.trk_max_iteration;
  a.huber = p.trk_lsnorm == ESVO_TRK_LSNORM_HUBER; a.huber_thr = p.trk_huber_threshold; a.analytical = analytical != 0;
  a.state = t->d.state;
  const int smem = (TRK_MAXB * 6 + TRK_MAXB * 2 + TRK_MAXB * 3 + 16 * 8) * 8;
  trk_solve_kernel<<<1, TRK_THREADS, smem, c->stream>>>(c->dc, a);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  double state[64];
  ESVO_CUDA_TRY(c, cudaMemcpyAsync(state, t->d.state, sizeof(state), cudaMemcpyDeviceToHost, c->stream));
  ESVO_CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  std::memcpy(Tout, state + 28, 128);
  if (st) { st->n_points = (int64_t)state[44]; st->nfev = (int64_t)state[45]; st->n_iter = (int64_t)state[46]; }
  return ESVO_OK;
}

ESVO_API int esvo_track_get_negative_ts(esvo_ctx* c, double* neg, double* du, double* dv) {
  CHECK_CTX(c);
  TrackState* t = c->trk;
  if (!t->ready) return ESVO_ERR_STATE;
  const DevConsts& dc = c->dc;
  const size_t npix = (size_t)dc.W * dc.H;
  std::vector<uint8_t> hn(npix); std::vector<int16_t> hu(npix), hv(npix);
  ESVO_CUDA_TRY(c, cudaMemcpy2D(hn.data(), dc.W, t->d.neg, dc.pitch, dc.W, dc.H, cudaMemcpyDeviceToHost));
  ESVO_CUDA_TRY(c, cudaMemcpy(hu.data(), t->d.du, npix * 2, cudaMemcpyDeviceToHost));
  ESVO_CUDA_TRY(c, cudaMemcpy(hv.data(), t->d.dv, npix * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < npix; ++i) { if (neg) neg[i] = hn[i]; if (du) du[i] = hu[i]; if (dv) dv[i] = hv[i]; }
  return ESVO_OK;
}

}  // extern "C"
