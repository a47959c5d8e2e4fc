// esvo_b200 product code -- per-seed inverse-depth refinement (sm_90a).
//
// Replaces esvo_core::core::DepthProblem::{operator(), warping, patchInterpolation}
// (esvo_core/src/core/DepthProblem.cpp:34-262), DepthProblemSolver::{solve,
// solve_multiple_problems, solve_single_problem_numerical, pointCulling}
// (esvo_core/src/core/DepthProblemSolver.cpp:28-244) and the pieces of Eigen's unsupported
// LevenbergMarquardt / NumericalDiff / covar that call site uses, specialised to one unknown.
//
// Design: one warp per seed runs the WHOLE 1-D Levenberg-Marquardt solve in registers, and the two 16-lane
// halves of the warp evaluate the residual vector at TWO inverse depths at once: half 0 at a point x, half 1 at
// x + h (h = NumericalDiff's forward step).  The LM driver always needs f at a trial point and, if the trial is
// accepted, f at trial + h for the next forward difference, so the second half is never idle: its result is
// either the next Jacobian column or (rejected trial) discarded speculation.  Within a half, lane l owns patch
// pixels l, l+16, l+32, ... (15x7 = 105 residuals -> 7 slots); a residual evaluation is 2 x 4 bilinear taps per
// pixel read straight from the u8 time surfaces (L1/L2 resident), the Student-t scale IRLS loop and all norms
// are 4-level xor-shuffle reductions that never leave the half.  With one unknown the QR factorisation collapses
// to  R = -sign(J_0)||J||,  Q^T f = J^T f / R, and lmpar/qrsolv to scalar Givens updates -- restated below
// statement by statement.  f64 throughout and no FMA contraction (-fmad=false) outside the explicit Newton
// refinements of the reciprocal / reciprocal square root.
// Algorithmic bytes per residual evaluation: 2 x 16 x 8 px x 4 B = 1024 B (SURVEY.md 8d).
#include <algorithm>

#include "common.cuh"

namespace esvo {

constexpr unsigned FULL = 0xffffffffu;

struct SeedGeom {   // lives in shared memory (warp-uniform, read once per evaluation)
  double coor0, coor1;
  double T[12];  // T_left_virtual (3x4)
};

struct LmArgs {
  const esvo_seed* seeds;
  const unsigned long long* n_ptr;  // device count (counters[1]) or null
  int n_fixed;
  const uint8_t *tl, *tr;
  double T_left_world[16];          // rigid inverse of the observation pose, by value (no upload, no pinned staging)
  int32_t* flag;
  double* res;                      // 3 per seed
  unsigned long long* counters;
};

// PerspectiveCamera::cam2World (CameraSystem.cpp:120-139) for P = [fx 0 cx tx; 0 fy cy ty; 0 0 1 tz]:
// solving [P; 0 0 0 z] p_s = [x y 1 1]^T gives p = ((x-cx-tx/z) z/fx, (y-cy-ty/z) z/fy, z (1 - tz/z)).
__device__ __forceinline__ void cam2world_dev(const DevConsts& dc, double x, double y, double rho, double p[3]) {
  const double z = 1.0 / rho;
  p[0] = (x - dc.cx - dc.Pl[3] / z) * z / dc.fx;
  p[1] = (y - dc.cy - dc.Pl[7] / z) * z / dc.fy;
  p[2] = z * (1.0 - dc.Pl[11] / z);
}

// Reductions over the 16 lanes of a half warp (xor offsets 8,4,2,1 never cross the halves); every lane of the
// half ends up with the half's total.  Must be called by all 32 lanes.
__device__ __forceinline__ double half_sum(double v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ int half_sum_i(int v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ double half_min(double v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(FULL, v, o));
  return v;
}
template <int S>
__device__ __forceinline__ double slot_tree_sum(const double (&t)[S]) {   // pairwise in-lane sum
  double u[S];
#pragma unroll
  for (int s = 0; s < S; ++s) u[s] = t[s];
#pragma unroll
  for (int w = 1; w < S; w <<= 1)
#pragma unroll
    for (int s = 0; s + w < S; s += 2 * w) u[s] += u[s + w];
  return u[0];
}

// DepthProblem::operator() (DepthProblem.cpp:34-160) for the inverse depth `rho` of THIS half warp.  off[s] is
// the lane's pixel offset (py*pitch+px) of slot s inside a patch, vmask its validity bits (k = hl+16s < N).
// fv[] receives the lane's residual slots (0 for padding).  Control flow is warp-uniform; everything that
// depends on rho is predicated, so the two halves stay converged around the shuffles.
// Sum over the lane's slots of a2/(nus + a2) with ONE reciprocal per group of up to four terms:
//   a/x + b/y = (a y + b x) / (x y),  (n01/p01) + (n23/p23) = (n01 p23 + n23 p01) / (p01 p23).
// All terms are >= 0 (no cancellation); every product stays far inside the normal range for nus > 1e-30
// (x <= 3e5, so p01 p23 <= 1e22; >= 1e-120).  Rounding-level deviation like the reciprocal form itself.
__device__ __forceinline__ double irls_group4(double a0, double a1, double a2, double a3, double nus) {
  const double d0 = nus + a0, d1 = nus + a1, d2 = nus + a2, d3 = nus + a3;
  const double p01 = d0 * d1, p23 = d2 * d3;
  const double n01 = fma(a0, d1, a1 * d0), n23 = fma(a2, d3, a3 * d2);
  return fma(n01, p23, n23 * p01) * rcp_nr(p01 * p23);
}
__device__ __forceinline__ double irls_group3(double a0, double a1, double a2, double nus) {
  const double d0 = nus + a0, d1 = nus + a1, d2 = nus + a2;
  const double p01 = d0 * d1;
  const double n01 = fma(a0, d1, a1 * d0);
  return fma(n01, d2, a2 * p01) * rcp_nr(p01 * d2);
}
__device__ __forceinline__ double irls_group2(double a0, double a1, double nus) {
  const double d0 = nus + a0, d1 = nus + a1;
  return fma(a0, d1, a1 * d0) * rcp_nr(d0 * d1);
}
// Degenerate regime of the reference's scale iteration (DepthProblem.cpp:96-119).  With m non-zero residuals of N the update
//   s' = (1/N) sum_i r_i^2 (nu+1) / (nu + r_i^2/s)  <=  s (nu+1) m / N = c s,
// so for c < 0.95 every exact step shrinks s by more than 5 %: s decays geometrically (thousands of passes) until r_i^2/s
// overflows to +inf for every pixel, the sum becomes exactly 0 and :116-119 resets the scale to td_scale^2.  That is only
// certain while rounding cannot pass the 5 % test: once s is subnormal (k steps of 2^-1074) a step's rounding error is below
// one step, so the loop can stall where 0.95 eps k <= 1 (eps = 1 - c / 0.95).  The smallest residual keeps the sum non-zero
// down to k = min r^2 / (DBL_MAX 2^-1074) = min r^2 / 2^-50, so the reset is proven when 0.95 eps min r^2 > 2^-50, i.e.
//   gap min r^2 > 2^-50 N  with gap = 0.95 N - (nu+1) m;
// the guard asks for twice that (DESIGN.md deviation 4).  The 1e-9 margin covers the rounding of steps at normal scales.
constexpr double kIrlsResetGap = 0x1p-49;
// r_min > 1e-6 alone proves the reset where gap >= kIrlsGapNoTiny N (eps >= 1.9e-3: every shipped shape at both shipped nu).
constexpr double kIrlsGapNoTiny = kIrlsResetGap / 1e-12;
__device__ __forceinline__ bool irls_degenerate(double nu1, int nz, int N) {
  return nu1 * (double)nz < 0.95 * (double)N * (1.0 - 1e-9);
}
__device__ __forceinline__ double irls_gap(double nu1, int nz, int N) { return 0.95 * (double)N - nu1 * (double)nz; }

template <int S>
__device__ __forceinline__ double irls_lane_sum(const double (&a)[S], double nus) {
  double acc = 0.0;
#pragma unroll
  for (int s = 0; s + 4 <= S; s += 4) acc += irls_group4(a[s], a[s + 1], a[s + 2], a[s + 3], nus);
  constexpr int R = S % 4, B = S - R;
  if (R == 3) acc += irls_group3(a[B], a[B + 1], a[B + 2], nus);
  if (R == 2) acc += irls_group2(a[B], a[B + 1], nus);
  if (R == 1) acc += a[B] * rcp_nr(nus + a[B]);
  return acc;
}

// TD: LSnorm is known to be Tdist at compile time (every shipped cfg) -- sheds the l2 / zncc code and registers.
template <int S, bool TD>
__device__ __forceinline__ void depth_residual_half(const DevConsts& dc, const SeedGeom& g, const uint8_t* __restrict__ tl,
                                                    const uint8_t* __restrict__ tr, double rho, const int (&off)[S], unsigned vmask,
                                                    double (&fv)[S]) {
  const int wx = dc.wx, wy = dc.wy, N = wx * wy, W = dc.W, H = dc.H;
  const int hx = (wx - 1) / 2, hy = (wy - 1) / 2;
  // ---- warping (:162-191) ----
  double p[3];
  cam2world_dev(dc, g.coor0, g.coor1, rho, p);
  double pl[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) pl[q] = g.T[q * 4 + 0] * p[0] + g.T[q * 4 + 1] * p[1] + g.T[q * 4 + 2] * p[2] + g.T[q * 4 + 3];
  double h1[3], h2[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    h1[q] = dc.Pl[q * 4 + 0] * pl[0] + dc.Pl[q * 4 + 1] * pl[1] + dc.Pl[q * 4 + 2] * pl[2] + dc.Pl[q * 4 + 3];
    h2[q] = dc.Pr[q * 4 + 0] * pl[0] + dc.Pr[q * 4 + 1] * pl[1] + dc.Pr[q * 4 + 2] * pl[2] + dc.Pr[q * 4 + 3];
  }
  const double x1 = h1[0] / h1[2], y1 = h1[1] / h1[2], x2 = h2[0] / h2[2], y2 = h2[1] / h2[2];
  bool ok = !(x1 < hx || x1 > W - hx || y1 < hy || y1 > H - hy) && !(x2 < hx || x2 > W - hx || y2 < hy || y2 > H - hy);
  // NaN coordinates (rho = 0 seeds): the reference's floor()->int conversion yields INT_MIN on x86 and the
  // patch is rejected at DepthProblem.cpp:204; make that explicit instead of relying on conversion UB.
  ok = ok && (x1 == x1) && (y1 == y1) && (x2 == x2) && (y2 == y2) && fabs(x1) < 1e9 && fabs(y1) < 1e9 && fabs(x2) < 1e9 && fabs(y2) < 1e9;
  // ---- patchInterpolation bounds (:193-239) for both images ----
  const double fx1 = floor(x1), fy1 = floor(y1), fx2 = floor(x2), fy2 = floor(y2);
  int ulx1 = 0, uly1 = 0, ulx2 = 0, uly2 = 0;
  if (ok) {
    ulx1 = (int)(fx1 - hx); uly1 = (int)(fy1 - hy); ulx2 = (int)(fx2 - hx); uly2 = (int)(fy2 - hy);
    const int drx1 = (int)(fx1 + hx), dry1 = (int)(fy1 + hy), drx2 = (int)(fx2 + hx), dry2 = (int)(fy2 + hy);
    ok = !(ulx1 < 0 || uly1 < 0 || drx1 >= W || dry1 >= H || uly1 + wy >= H || ulx1 + wx >= W) &&
         !(ulx2 < 0 || uly2 < 0 || drx2 >= W || dry2 >= H || uly2 + wy >= H || ulx2 + wx >= W);
  }
  if (!ok) { ulx1 = uly1 = ulx2 = uly2 = 0; }   // a failed half still walks a (valid) dummy patch: no divergence
  // bilinear weights (:215-223)
  const double q1a = (fx1 + 1) - x1, q2a = x1 - fx1, q3a = (fy1 + 1) - y1, q4a = y1 - fy1;
  const double q1b = (fx2 + 1) - x2, q2b = x2 - fx2, q3b = (fy2 + 1) - y2, q4b = y2 - fy2;
  const uint8_t* basea = tl + (size_t)uly1 * dc.pitch + ulx1;
  const uint8_t* baseb = tr + (size_t)uly2 * dc.pitch + ulx2;
  double r[S], t1v[S];
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const uint8_t* pa = basea + off[s];
    const uint8_t* pb = baseb + off[s];
    const double a00 = pa[0], a01 = pa[1], a10 = pa[dc.pitch], a11 = pa[dc.pitch + 1];
    const double b00 = pb[0], b01 = pb[1], b10 = pb[dc.pitch], b11 = pb[dc.pitch + 1];
    const double t1 = q3a * (q1a * a00 + q2a * a01) + q4a * (q1a * a10 + q2a * a11);   // (:253-259)
    const double t2 = q3b * (q1b * b00 + q2b * b01) + q4b * (q1b * b10 + q2b * b11);
    const bool on = ok && ((vmask >> s) & 1u);
    r[s] = on ? t1 - t2 : 0.0;
    if (!TD && dc.lsnorm == ESVO_LSNORM_ZNCC) { t1v[s] = on ? t1 : 0.0; r[s] = on ? t2 : 0.0; }   // zncc needs both patches (rare path)
  }
  // ---- constant failure residual (:40-58, :140-157) ----
  double failval;
  if (!TD && dc.lsnorm == ESVO_LSNORM_L2) failval = 255.0;
  else if (!TD && dc.lsnorm == ESVO_LSNORM_ZNCC) failval = 2.0 / sqrt((double)N);
  else { const double q = 255.0 / dc.td_scale; failval = sqrt((dc.td_nu + 1) / (dc.td_nu + q * q)) * 255.0; }

  if (!TD && dc.lsnorm == ESVO_LSNORM_L2) {
#pragma unroll
    for (int s = 0; s < S; ++s) fv[s] = ((vmask >> s) & 1u) ? (ok ? r[s] : failval) : 0.0;
    return;
  }
  if (!TD && dc.lsnorm == ESVO_LSNORM_ZNCC) {
    double m1 = 0, m2 = 0;   // t1 in t1v[], t2 in r[]
#pragma unroll
    for (int s = 0; s < S; ++s) { m1 += t1v[s]; m2 += r[s]; }
    m1 = half_sum(m1) / N; m2 = half_sum(m2) / N;
    double s1 = 0, s2 = 0;
#pragma unroll
    for (int s = 0; s < S; ++s)
      if ((vmask >> s) & 1u) { s1 += (t1v[s] - m1) * (t1v[s] - m1); s2 += (r[s] - m2) * (r[s] - m2); }
    s1 = sqrt(half_sum(s1) / N) + 1e-6; s2 = sqrt(half_sum(s2) / N) + 1e-6;
#pragma unroll
    for (int s = 0; s < S; ++s) {
      const double z = ((t1v[s] - m1) / s1 - (r[s] - m2) / s2) / sqrt((double)N);
      fv[s] = ((vmask >> s) & 1u) ? (ok ? z : failval) : 0.0;
    }
    return;
  }
  // ---- Student-t: IRLS on the scale (:89-135) ----
  // r[s] is exactly 0 for padding, failed halves and zero residuals, so a2 = r^2 contributes exactly 0 to every
  // sum below -- the same as being skipped by :112.
  double a2[S];
  int nz = 0;
  double rmin = 1e300;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    a2[s] = r[s] * r[s];
    if (r[s] != 0) { nz++; rmin = fmin(rmin, fabs(r[s])); }
  }
  // Degenerate regime (irls_degenerate): jump straight to the reset where it is proven.
  nz = half_sum_i(nz);
  rmin = half_min(rmin);
  const double nu1 = dc.td_nu + 1, invN = 1.0 / (double)N;
  double sc1 = dc.td_scale2, sc2 = -1.0;
  bool run = ok;
  if (run && irls_degenerate(nu1, nz, N) && irls_gap(nu1, nz, N) * (rmin * rmin) >= kIrlsResetGap * (double)N) {
    sc2 = dc.td_scale2; run = false;
  }
  // Fast loop: both halves iterate together (a finished half keeps computing, its updates are masked).
  // sum_i r_i^2 (nu+1) / (nu + r_i^2/s) == (nu+1) s sum_i a2_i / (nu s + a2_i), one reciprocal per four pixels.
  while (__any_sync(FULL, run && sc1 > 1e-30)) {
    const double nus = dc.td_nu * sc1, c1 = nu1 * sc1;
    const double sum = c1 * half_sum(irls_lane_sum<S>(a2, nus));
    if (run && sc1 > 1e-30) {
      if (sum == 0) { sc2 = dc.td_scale2; run = false; }
      else {
        sc2 = sum * invN;
        run = fabs(sc2 - sc1) > 0.05 * sc1;
        sc1 = sc2;
      }
    }
  }
  // r^2 (nu+1) / (nu + r^2/s) == (r^2 (nu+1) s) / (nu s + r^2): one reciprocal per pixel, S independent chains.
  // Only the rare scales below 1e-30 get here.
  while (__any_sync(FULL, run && sc1 > 1e-250)) {
    const double nus = dc.td_nu * sc1, c1 = nu1 * sc1;
    double t[S];
#pragma unroll
    for (int s = 0; s < S; ++s) t[s] = (a2[s] * c1) * rcp_nr(nus + a2[s]);
    const double sum = half_sum(slot_tree_sum<S>(t));
    if (run && sc1 > 1e-250) {
      if (sum == 0) { sc2 = dc.td_scale2; run = false; }
      else {
        sc2 = sum * invN;
        run = fabs(sc2 - sc1) > 0.05 * sc1;      // loop test of :96 without the division
        sc1 = sc2;
      }
    }
  }
  // Denormal corner (scale decayed below 1e-250 without the shortcut applying): plain divisions, exact semantics.
  while (__any_sync(FULL, run)) {
    double sum = 0;
#pragma unroll
    for (int s = 0; s < S; ++s) if (a2[s] != 0) sum += a2[s] * (nu1 / (dc.td_nu + a2[s] / sc1));
    sum = half_sum(sum);
    if (run) {
      if (sum == 0) { sc2 = dc.td_scale2; run = false; }
      else { sc2 = sum * invN; run = fabs(sc2 - sc1) / sc1 > 0.05; sc1 = sc2; }
    }
  }
  // weights (:121-133): sqrt((nu+1)/(nu + r^2/s)) r == r sqrt((nu+1) s) / sqrt(nu s + r^2)
  const bool tiny = __any_sync(FULL, ok && !(sc2 > 1e-200));
  if (!tiny) {
    const double sc = ok ? sc2 : 1.0;
    const double nus = dc.td_nu * sc, k1 = sqrt_nr(nu1 * sc);
#pragma unroll
    for (int s = 0; s < S; ++s) {
      const double f = r[s] * (k1 * rsqrt_nr(nus + a2[s]));
      fv[s] = ((vmask >> s) & 1u) ? (ok ? f : failval) : 0.0;
    }
  } else {
#pragma unroll
    for (int s = 0; s < S; ++s) {
      const double w = nu1 / (dc.td_nu + a2[s] / sc2);
      fv[s] = ((vmask >> s) & 1u) ? (ok ? sqrt(w) * r[s] : failval) : 0.0;
    }
  }
}

// Eigen JacobiRotation::makeGivens (real)
__device__ __forceinline__ void make_givens(double p, double q, double& c, double& s) {
  if (q == 0) { c = p < 0 ? -1 : 1; s = 0; }
  else if (p == 0) { c = 0; s = q < 0 ? 1 : -1; }
  else if (fabs(p) > fabs(q)) { double t = q / p, u = sqrt(1 + t * t); if (p < 0) u = -u; c = 1 / u; s = -t * c; }
  else { double t = p / q, u = sqrt(1 + t * t); if (q < 0) u = -u; s = -1 / u; c = -t * s; }
}

// internal::lmpar2 + qrsolv for n = 1 (R = r, qtb = q, diag = d).  Returns x; updates par.
__device__ __noinline__ double lmpar_1d(double r, double d, double q, double delta, double& par) {
  const double dwarf = 2.2250738585072014e-308;
  // rank is 1 here (callers guarantee r != 0)
  double x = q / r;
  double dxnorm = fabs(d * x);
  double fp = dxnorm - delta;
  if (fp <= 0.1 * delta) { par = 0; return x; }
  double parl;
  { double w = d * (d * x) / dxnorm; w = w / r; double temp = fabs(w); parl = fp / delta / temp / temp; }
  double gnorm = fabs(r * q / d);
  double paru = gnorm / delta;
  if (paru == 0.) paru = dwarf / fmin(delta, 0.1);
  par = fmax(par, parl);
  par = fmin(par, paru);
  if (par == 0.) par = gnorm / dxnorm;
  int iter = 0;
  while (true) {
    ++iter;
    if (par == 0.) par = fmax(dwarf, .001 * paru);
    const double sd = sqrt(par) * d;     // wa1 = sqrt(par)*diag
    double c, s;
    make_givens(-r, sd, c, s);           // qrsolv, one rotation
    const double rr = c * r + s * sd;    // modified diagonal element
    const double wa = c * q + s * 0.0;   // (q^T b, 0) component
    x = wa / rr;
    dxnorm = fabs(d * x);
    double temp = fp;
    fp = dxnorm - delta;
    if (fabs(fp) <= 0.1 * delta || (parl == 0. && fp <= temp && temp < 0.) || iter == 10) break;
    double w = d * ((d * x) / dxnorm);
    w /= rr;
    temp = fabs(w);
    const double parc = fp / delta / temp / temp;
    if (fp > 0.) parl = fmax(parl, par);
    if (fp < 0.) paru = fmin(paru, par);
    par = fmax(parl, par + parc);
  }
  return x;
}

// S = residual slots per lane: 7 covers patches up to 112 pixels (the shipped 15x7), 8 up to kMaxPatch = 128.
template <int S, bool TD>
__global__ void __launch_bounds__(32, 16) lm_kernel(DevConsts dc, LmArgs a) {
  const int lane = threadIdx.x & 31, half = lane >> 4, hl = lane & 15;
  const int k = blockIdx.x;
  const int n = a.n_ptr ? (int)*a.n_ptr : a.n_fixed;
  if (k >= n) return;
  const esvo_seed& sd = a.seeds[k];
  const int m = dc.wx * dc.wy;
  // Cold per-seed state is kept in shared memory so that the hot loops fit the register budget of MB seeds / SM:
  // the patch geometry (warp-uniform) and fcur, the accepted residual vectors (touched once per LM step).
  __shared__ SeedGeom g;
  __shared__ double s_fcur[S][32];
  // setProblem (:17-32): T_left_virtual = T_left_world * T_world_virtual (top 3 rows); lane q computes entry q
  if (lane < 12) {
    const int r = lane >> 2, cidx = lane & 3;
    double s = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += a.T_left_world[r * 4 + j] * sd.T_world_virtual[j * 4 + cidx];
    g.T[lane] = s;
  } else if (lane == 12) { g.coor0 = sd.x_left[0]; g.coor1 = sd.x_left[1]; }
  __syncwarp();
  // the lane's pixels inside a patch: k = hl + 16 s  ->  (py, px) = (k / wx, k % wx)
  int off[S];
  unsigned vmask = 0;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const int kk = hl + 16 * s;
    const bool v = kk < m;
    const int py = kk / dc.wx, px = kk - py * dc.wx;
    off[s] = v ? py * dc.pitch + px : 0;
    vmask |= (v ? 1u : 0u) << s;
  }
  const double EPS = 2.220446049250313e-16;
  const double ftol = 1e-6, xtol = 1e-6, factor = 100.;
  const int maxfev = dc.max_iter * 3;
  double x = sd.inv_depth;
  const double HEPS = 1.4901161193847656e-08;   // sqrt(DBL_EPSILON), NumericalDiff's step factor
  // s_fcur[.][lane] -- half 0: f(x), half 1: f(x+h) with h = HEPS*|x|, for the lane's pixels
  double fnew[S];
  auto hstep = [&](double xx) { double h = HEPS * fabs(xx); return h == 0. ? HEPS : h; };
  // The solver is written as a small state machine around ONE call site of the (large, fully inlined)
  // residual evaluation, which keeps the kernel's instruction footprint -- and its I-cache misses -- low:
  //   phase 0: evaluate {x, x+h}                  (minimizeInit + the first forward-difference point)
  //   phase 1: evaluate {trial, trial+h(trial)}   (inside minimizeOneStep's do-while; the second point is
  //            speculative: it becomes f(x+h) of the next step if the trial is accepted)
  int nfev = 0, nexec = 0;
  double fnorm = 0, par = 0.; int iter = 1;
  double diag = 0, delta = 0, xnorm = 0, r00 = 0, qtf = 0, gnorm = 0;
  double xn = x, pstep = 0, pnorm = 0;
  int iteration = 0, optState = 0;
  int phase = 0;
  bool done = false;
  // The (warp-uniform) solver state is parked in shared memory across the residual evaluation, the only place
  // where register pressure matters; every lane holds identical values, lane 0 writes them.
  __shared__ double s_st[12];
  __shared__ int s_si[6];
  while (!done) {
    const double xe = (phase == 0) ? x : xn;
    const double rho_e = half ? xe + hstep(xe) : xe;
    if (lane == 0) {
      s_st[0] = x; s_st[1] = xn; s_st[2] = fnorm; s_st[3] = par; s_st[4] = diag; s_st[5] = delta; s_st[6] = xnorm;
      s_st[7] = r00; s_st[8] = qtf; s_st[9] = gnorm; s_st[10] = pstep; s_st[11] = pnorm;
      s_si[0] = nfev; s_si[1] = nexec; s_si[2] = iter; s_si[3] = iteration; s_si[4] = optState; s_si[5] = phase;
    }
    __syncwarp();
    depth_residual_half<S, TD>(dc, g, a.tl, a.tr, rho_e, off, vmask, fnew);
    __syncwarp();
    x = s_st[0]; xn = s_st[1]; fnorm = s_st[2]; par = s_st[3]; diag = s_st[4]; delta = s_st[5]; xnorm = s_st[6];
    r00 = s_st[7]; qtf = s_st[8]; gnorm = s_st[9]; pstep = s_st[10]; pnorm = s_st[11];
    nfev = s_si[0]; nexec = s_si[1]; iter = s_si[2]; iteration = s_si[3]; optState = s_si[4]; phase = s_si[5];
    double ss = 0;
#pragma unroll
    for (int s = 0; s < S; ++s) ss += fnew[s] * fnew[s];
    const double fn_new = sqrt(__shfl_sync(FULL, half_sum(ss), 0));   // ||f(xe)||: half 0's total
    bool step_finished;          // does control fall through to "begin the next minimizeOneStep"?
    if (phase == 0) {
      // ---- minimizeInit ----
      nfev = 1; nexec = 2;
#pragma unroll
      for (int s = 0; s < S; ++s) s_fcur[s][lane] = fnew[s];
      fnorm = fn_new;
      par = 0.; iter = 1;
      step_finished = true;      // go and start the first step
    } else {
      // ---- body of minimizeOneStep's do-while after the trial evaluation ----
      ++nfev; ++nexec;
      int status = -1;
      const double fnorm1 = fn_new;
      double actred = -1.;
      if (.1 * fnorm1 < fnorm) actred = 1. - (fnorm1 / fnorm) * (fnorm1 / fnorm);
      const double t1 = fabs(r00 * pstep) / fnorm, temp1 = t1 * t1;
      const double t2 = sqrt(par) * pnorm / fnorm, temp2 = t2 * t2;
      const double prered = temp1 + temp2 / .5;
      const double dirder = -(temp1 + temp2);
      double ratio = 0.;
      if (prered != 0.) ratio = actred / prered;
      if (ratio <= .25) {
        double temp = 0;
        if (actred >= 0.) temp = .5;
        if (actred < 0.) temp = .5 * dirder / (dirder + .5 * actred);
        if (.1 * fnorm1 >= fnorm || temp < .1) temp = .1;
        delta = temp * fmin(delta, pnorm / .1);
        par /= temp;
      } else if (!(par != 0. && ratio < .75)) {
        delta = pnorm / .5;
        par = .5 * par;
      }
      if (ratio >= 1e-4) {
        x = xn;
#pragma unroll
        for (int s = 0; s < S; ++s) s_fcur[s][lane] = fnew[s];
        ++nexec;   // the speculative f(x+h) is consumed by the next step
        xnorm = fabs(diag * x);
        fnorm = fnorm1;
        ++iter;
      }
      if (fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1. && delta <= xtol * xnorm) status = 3;
      else if (fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1.) status = 1;
      else if (delta <= xtol * xnorm) status = 2;
      else if (nfev >= maxfev) status = 5;
      else if (fabs(actred) <= EPS && prered <= EPS && .5 * ratio <= 1.) status = 6;
      else if (delta <= EPS * xnorm) status = 7;
      else if (gnorm <= EPS) status = 8;
      if (status == -1 && ratio < 1e-4) {
        // unsuccessful trial: stay inside the do-while with the updated trust region
        pstep = -lmpar_1d(r00, diag, qtf, delta, par);
        xn = x + pstep;
        pnorm = fabs(diag * pstep);
        if (iter == 1) delta = fmin(delta, pnorm);
        continue;
      }
      // ---- DepthProblemSolver loop control (:165-186) ----
      iteration++;
      if (iteration >= dc.max_iter) { done = true; continue; }
      if (status == 2 || status == 3) { if (optState == 0) optState++; else { done = true; continue; } }
      step_finished = true;
    }
    // ================= begin minimizeOneStep (repeats without evaluation while it returns CosinusTooSmall) =========
    while (step_finished && !done) {
      // NumericalDiff<Forward>::df: the reference evaluates f(x) again and then f(x+h); both are already
      // known here (the two halves of fcur), we only account for them in nfev.
      const double h = hstep(x);
      nfev += 2;
      double jj = 0, jf = 0, j0 = 0;
      __syncwarp();
#pragma unroll
      for (int s = 0; s < S; ++s) {
        const double f0 = s_fcur[s][hl], f1 = s_fcur[s][hl + 16];   // f(x), f(x+h) of this pixel
        const double J = div_nr(f1 - f0, h);
        if (s == 0) j0 = J;
        jj += J * J; jf += J * f0;
      }
      __syncwarp();
      jj = half_sum(jj); jf = half_sum(jf);            // identical in both halves
      j0 = __shfl_sync(FULL, j0, 0);
      const double wa2 = sqrt(jj);
      // ColPivHouseholderQR of a single column: R00 = -sign(J0)*||J|| (beta), unless the tail is zero
      r00 = (j0 >= 0) ? -wa2 : wa2;
      if (iter == 1) {
        diag = (wa2 == 0.) ? 1. : wa2;
        xnorm = fabs(diag * x);
        delta = factor * xnorm;
        if (delta == 0.) delta = factor;
      }
      qtf = (wa2 != 0.) ? jf / r00 : 0.0;
      gnorm = 0.;
      if (fnorm != 0. && wa2 != 0.) gnorm = fabs(r00 * (qtf / fnorm)) / wa2;
      if (gnorm <= 0.) {
        // CosinusTooSmall (gtol = 0): the step returns at once; the solver loop calls it again
        iteration++;
        if (iteration >= dc.max_iter) done = true;
        continue;
      }
      diag = fmax(diag, wa2);
      pstep = -lmpar_1d(r00, diag, qtf, delta, par);
      xn = x + pstep;
      pnorm = fabs(diag * pstep);
      if (iter == 1) delta = fmin(delta, pnorm);
      phase = 1;
      step_finished = false;     // a trial evaluation is needed
    }
  }
  if (lane == 0) {
    atomicAdd(&a.counters[6], (unsigned long long)nfev);
    atomicAdd(&a.counters[7], (unsigned long long)nexec);
    int ok = !(x <= 0.001);                                               // :192
    double var = 0.0;
    const double inv = (r00 != 0.) ? (1. / r00) * (1. / r00) : 0.0;       // internal::covar, n = 1
    if (!TD && dc.lsnorm == ESVO_LSNORM_L2) var = (fnorm * fnorm / (m - 1)) * inv;   // :200-206
    else var = (dc.td_stdvar * dc.td_stdvar) * inv;                       // :207-211 (Tdist; zncc leaves it unset)
    a.flag[k] = ok;
    a.res[3 * k] = x; a.res[3 * k + 1] = var; a.res[3 * k + 2] = fnorm * fnorm;      // :212
  }
}

// --------------------------------------------------------------------------------------------
// lm2_kernel: the same solver (same arithmetic, same order of every floating-point operation as lm_kernel with
// TD = true, IRLS = 1) reorganised around the instruction stream.  A saturated launch of lm_kernel stalls first on
// instruction fetch (`no_instructions`): every evaluation walks
// ~2 200 straight-line instructions (7 unrolled patch slots x bilinear taps / weights / Jacobian terms) exactly once,
// so the 16-24 warps of an SM, all at different places of a 70 KB kernel, stream code through the instruction caches.
// Here the per-slot phases are ROLLED loops (7 trips of ~60 / ~35 / ~25 instructions) that hand their per-lane values
// over through shared memory (residuals r, the two residual vectors f(x) | f(x+h) double-buffered); only the scale
// iteration keeps its seven squared residuals in registers.  Register pressure drops with it (no parking of the
// solver state needed), so more seeds are resident per SM.  The bilinear taps are per-lane LDG.E.U8 against L1 (97 % hit
// rate); staging the source tiles in shared memory by TMA gained nothing (DESIGN.md §9).
// --------------------------------------------------------------------------------------------
template <int S, int MB>
__global__ void __launch_bounds__(32, MB) lm2_kernel(DevConsts dc, LmArgs a) {
  const int lane = threadIdx.x & 31, half = lane >> 4, hl = lane & 15;
  const int k = blockIdx.x;
  const int n = a.n_ptr ? (int)*a.n_ptr : a.n_fixed;
  if (k >= n) return;
  const esvo_seed& sd = a.seeds[k];
  const int wx = dc.wx, wy = dc.wy, m = wx * wy, W = dc.W, H = dc.H;
  const int hx = (wx - 1) / 2, hy = (wy - 1) / 2;
  const int n_valid = m > hl ? (m - hl + 15) / 16 : 0;   // the lane's slots 0 .. n_valid-1 hold patch pixels (hl + 16 s < m)
  __shared__ SeedGeom g;
  __shared__ int s_off[S * 16];
  __shared__ double s_r[S][32];
  __shared__ double s_f[2][S][32];
  if (lane < 12) {
    const int r = lane >> 2, cidx = lane & 3;
    double s = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += a.T_left_world[r * 4 + j] * sd.T_world_virtual[j * 4 + cidx];
    g.T[lane] = s;
  } else if (lane == 12) { g.coor0 = sd.x_left[0]; g.coor1 = sd.x_left[1]; }
  // pixel offsets of the lane's slots: kk = hl + 16 s -> (py, px) = (kk / wx, kk % wx); the same for both halves
  for (int q = lane; q < S * 16; q += 32) {
    const int s = q >> 4, kk = (q & 15) + 16 * s;
    const int py = kk / wx, px = kk - py * wx;
    s_off[q] = kk < m ? py * dc.pitch + px : 0;
  }
  __syncwarp();
  const double EPS = 2.220446049250313e-16;
  const double ftol = 1e-6, xtol = 1e-6, factor = 100.;
  const int maxfev = dc.max_iter * 3;
  const double HEPS = 1.4901161193847656e-08;
  auto hstep = [&](double xx) { double h = HEPS * fabs(xx); return h == 0. ? HEPS : h; };
  const double nu = dc.td_nu, nu1 = dc.td_nu + 1, invN = 1.0 / (double)m;
  double failval;
  { const double q = 255.0 / dc.td_scale; failval = sqrt((dc.td_nu + 1) / (dc.td_nu + q * q)) * 255.0; }

  double x = sd.inv_depth;
  int nfev = 0, nexec = 0;
  double fnorm = 0, par = 0.; int iter = 1;
  double diag = 0, delta = 0, xnorm = 0, r00 = 0, qtf = 0, gnorm = 0;
  double xn = x, pstep = 0, pnorm = 0;
  int iteration = 0, optState = 0;
  int phase = 0, cur = 0;       // cur: which s_f buffer holds the accepted f(x) | f(x+h)
  bool done = false;
  while (!done) {
    const double xe = (phase == 0) ? x : xn;
    const double rho = half ? xe + hstep(xe) : xe;
    const int nb = (phase == 0) ? 0 : 1 - cur;   // buffer this evaluation writes
    // ================= DepthProblem::operator() for this half's rho (DepthProblem.cpp:34-160) =================
    bool ok;
    int nz = 0;
    bool tiny = false;            // a non-zero residual of magnitude <= 1e-6 (the only thing the minimum was needed for)
    {
      double p[3];
      cam2world_dev(dc, g.coor0, g.coor1, rho, p);
      double pl[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) pl[q] = g.T[q * 4 + 0] * p[0] + g.T[q * 4 + 1] * p[1] + g.T[q * 4 + 2] * p[2] + g.T[q * 4 + 3];
      double h1[3], h2[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        h1[q] = dc.Pl[q * 4 + 0] * pl[0] + dc.Pl[q * 4 + 1] * pl[1] + dc.Pl[q * 4 + 2] * pl[2] + dc.Pl[q * 4 + 3];
        h2[q] = dc.Pr[q * 4 + 0] * pl[0] + dc.Pr[q * 4 + 1] * pl[1] + dc.Pr[q * 4 + 2] * pl[2] + dc.Pr[q * 4 + 3];
      }
      const double x1 = h1[0] / h1[2], y1 = h1[1] / h1[2], x2 = h2[0] / h2[2], y2 = h2[1] / h2[2];
      ok = !(x1 < hx || x1 > W - hx || y1 < hy || y1 > H - hy) && !(x2 < hx || x2 > W - hx || y2 < hy || y2 > H - hy);
      ok = ok && (x1 == x1) && (y1 == y1) && (x2 == x2) && (y2 == y2) && fabs(x1) < 1e9 && fabs(y1) < 1e9 && fabs(x2) < 1e9 && fabs(y2) < 1e9;
      const double fx1 = floor(x1), fy1 = floor(y1), fx2 = floor(x2), fy2 = floor(y2);
      int ulx1 = 0, uly1 = 0, ulx2 = 0, uly2 = 0;
      if (ok) {
        ulx1 = (int)(fx1 - hx); uly1 = (int)(fy1 - hy); ulx2 = (int)(fx2 - hx); uly2 = (int)(fy2 - hy);
        const int drx1 = (int)(fx1 + hx), dry1 = (int)(fy1 + hy), drx2 = (int)(fx2 + hx), dry2 = (int)(fy2 + hy);
        ok = !(ulx1 < 0 || uly1 < 0 || drx1 >= W || dry1 >= H || uly1 + wy >= H || ulx1 + wx >= W) &&
             !(ulx2 < 0 || uly2 < 0 || drx2 >= W || dry2 >= H || uly2 + wy >= H || ulx2 + wx >= W);
      }
      if (!ok) { ulx1 = uly1 = ulx2 = uly2 = 0; }
      const double q1a = (fx1 + 1) - x1, q2a = x1 - fx1, q3a = (fy1 + 1) - y1, q4a = y1 - fy1;
      const double q1b = (fx2 + 1) - x2, q2b = x2 - fx2, q3b = (fy2 + 1) - y2, q4b = y2 - fy2;
      const uint8_t* basea = a.tl + (size_t)uly1 * dc.pitch + ulx1;
      const uint8_t* baseb = a.tr + (size_t)uly2 * dc.pitch + ulx2;
      // ---- phase A: residuals of the lane's slots (rolled) ----
#pragma unroll 1
      for (int s = 0; s < S; ++s) {
        const int o = s_off[s * 16 + hl];
        const uint8_t* pa = basea + o;
        const uint8_t* pb = baseb + o;
        const double a00 = pa[0], a01 = pa[1], a10 = pa[dc.pitch], a11 = pa[dc.pitch + 1];
        const double b00 = pb[0], b01 = pb[1], b10 = pb[dc.pitch], b11 = pb[dc.pitch + 1];
        const double t1 = q3a * (q1a * a00 + q2a * a01) + q4a * (q1a * a10 + q2a * a11);
        const double t2 = q3b * (q1b * b00 + q2b * b01) + q4b * (q1b * b10 + q2b * b11);
        const bool on = ok && (s < n_valid);
        const double r = on ? t1 - t2 : 0.0;
        s_r[s][lane] = r;
        if (r != 0) { nz++; tiny |= fabs(r) <= 1e-6; }
      }
    }
    // ---- phase B: Student-t scale iteration (:89-135), squared residuals in registers ----
    double sc2 = -1.0;
    {
      double a2[S];
#pragma unroll
      for (int s = 0; s < S; ++s) { const double r = s_r[s][lane]; a2[s] = r * r; }
      nz = half_sum_i(nz);
      // Degenerate regime (irls_degenerate).  Far from the 0.95 threshold r_min > 1e-6 proves the reset; closer to it the half
      // needs min r^2 itself.  Such a half votes with all its lanes, so one ballot serves both and the min reduction runs
      // only when some half shows all 16 lanes set.
      const bool deg = irls_degenerate(nu1, nz, m);
      const double gap = irls_gap(nu1, nz, m);
      const bool need_min = ok && deg && gap < kIrlsGapNoTiny * (double)m;
      const unsigned vote = __ballot_sync(FULL, tiny || need_min);
      const bool no_tiny = ((vote >> (half * 16)) & 0xffffu) == 0;      // min |r| over the non-zero residuals > 1e-6
      double a2min = 1e300;
      if ((vote & 0xffffu) == 0xffffu || (vote >> 16) == 0xffffu) {   // warp-uniform
#pragma unroll
        for (int s = 0; s < S; ++s) if (a2[s] != 0) a2min = fmin(a2min, a2[s]);
        a2min = half_min(a2min);
      }
      double sc1 = dc.td_scale2;
      bool run = ok;
      if (run && deg && (need_min ? gap * a2min >= kIrlsResetGap * (double)m : no_tiny)) { sc2 = dc.td_scale2; run = false; }
      while (__any_sync(FULL, run && sc1 > 1e-30)) {
        const double nus = nu * sc1, c1 = nu1 * sc1;
        const double sum = c1 * half_sum(irls_lane_sum<S>(a2, nus));
        if (run && sc1 > 1e-30) {
          if (sum == 0) { sc2 = dc.td_scale2; run = false; }
          else { sc2 = sum * invN; run = fabs(sc2 - sc1) > 0.05 * sc1; sc1 = sc2; }
        }
      }
      // rare: scale below 1e-30 (one reciprocal per pixel), then the denormal corner with plain divisions
      while (__any_sync(FULL, run && sc1 > 1e-250)) {
        const double nus = nu * sc1, c1 = nu1 * sc1;
        double t[S];
#pragma unroll
        for (int s = 0; s < S; ++s) t[s] = (a2[s] * c1) * rcp_nr(nus + a2[s]);
        const double sum = half_sum(slot_tree_sum<S>(t));
        if (run && sc1 > 1e-250) {
          if (sum == 0) { sc2 = dc.td_scale2; run = false; }
          else { sc2 = sum * invN; run = fabs(sc2 - sc1) > 0.05 * sc1; sc1 = sc2; }
        }
      }
      while (__any_sync(FULL, run)) {
        double sum = 0;
#pragma unroll
        for (int s = 0; s < S; ++s) if (a2[s] != 0) sum += a2[s] * (nu1 / (nu + a2[s] / sc1));
        sum = half_sum(sum);
        if (run) {
          if (sum == 0) { sc2 = dc.td_scale2; run = false; }
          else { sc2 = sum * invN; run = fabs(sc2 - sc1) / sc1 > 0.05; sc1 = sc2; }
        }
      }
    }
    // ---- phase C: weighted residuals (:121-133) into the new buffer, their squared norm on the way (rolled) ----
    double ss = 0;
    {
      const bool tiny = __any_sync(FULL, ok && !(sc2 > 1e-200));
      const double sc = ok ? sc2 : 1.0;
      const double nus = nu * sc, k1 = tiny ? 0.0 : sqrt_nr(nu1 * sc);
      const double* pr = &s_r[0][lane];
      double* pf = &s_f[nb][0][lane];
#pragma unroll 1
      for (int s = 0; s < S; ++s, pr += 32, pf += 32) {
        const double r = *pr, a2v = r * r;
        double f;
        if (!tiny) f = r * (k1 * rsqrt_nr(nus + a2v));
        else f = sqrt(nu1 / (nu + a2v / sc2)) * r;
        const double fv = (s < n_valid) ? (ok ? f : failval) : 0.0;
        *pf = fv;
        ss += fv * fv;
      }
    }
    __syncwarp();
    const double fn_new = sqrt(__shfl_sync(FULL, half_sum(ss), 0));   // ||f(xe)||: half 0's total
    bool step_finished;
    if (phase == 0) {
      nfev = 1; nexec = 2;
      cur = 0;
      fnorm = fn_new;
      par = 0.; iter = 1;
      step_finished = true;
    } else {
      ++nfev; ++nexec;
      int status = -1;
      const double fnorm1 = fn_new;
      double actred = -1.;
      if (.1 * fnorm1 < fnorm) actred = 1. - (fnorm1 / fnorm) * (fnorm1 / fnorm);
      const double t1 = fabs(r00 * pstep) / fnorm, temp1 = t1 * t1;
      const double t2 = sqrt(par) * pnorm / fnorm, temp2 = t2 * t2;
      const double prered = temp1 + temp2 / .5;
      const double dirder = -(temp1 + temp2);
      double ratio = 0.;
      if (prered != 0.) ratio = actred / prered;
      if (ratio <= .25) {
        double temp = 0;
        if (actred >= 0.) temp = .5;
        if (actred < 0.) temp = .5 * dirder / (dirder + .5 * actred);
        if (.1 * fnorm1 >= fnorm || temp < .1) temp = .1;
        delta = temp * fmin(delta, pnorm / .1);
        par /= temp;
      } else if (!(par != 0. && ratio < .75)) {
        delta = pnorm / .5;
        par = .5 * par;
      }
      if (ratio >= 1e-4) {
        x = xn;
        cur = nb;
        ++nexec;
        xnorm = fabs(diag * x);
        fnorm = fnorm1;
        ++iter;
      }
      if (fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1. && delta <= xtol * xnorm) status = 3;
      else if (fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1.) status = 1;
      else if (delta <= xtol * xnorm) status = 2;
      else if (nfev >= maxfev) status = 5;
      else if (fabs(actred) <= EPS && prered <= EPS && .5 * ratio <= 1.) status = 6;
      else if (delta <= EPS * xnorm) status = 7;
      else if (gnorm <= EPS) status = 8;
      if (status == -1 && ratio < 1e-4) {
        pstep = -lmpar_1d(r00, diag, qtf, delta, par);
        xn = x + pstep;
        pnorm = fabs(diag * pstep);
        if (iter == 1) delta = fmin(delta, pnorm);
        continue;
      }
      iteration++;
      if (iteration >= dc.max_iter) { done = true; continue; }
      if (status == 2 || status == 3) { if (optState == 0) optState++; else { done = true; continue; } }
      step_finished = true;
    }
    while (step_finished && !done) {
      const double h = hstep(x);
      nfev += 2;
      double jj = 0, jf = 0, j0 = 0;
#pragma unroll 1
      for (int s = 0; s < S; ++s) {
        const double f0 = s_f[cur][s][hl], f1 = s_f[cur][s][hl + 16];
        const double J = div_nr(f1 - f0, h);
        if (s == 0) j0 = J;
        jj += J * J; jf += J * f0;
      }
      jj = half_sum(jj); jf = half_sum(jf);
      j0 = __shfl_sync(FULL, j0, 0);
      const double wa2 = sqrt(jj);
      r00 = (j0 >= 0) ? -wa2 : wa2;
      if (iter == 1) {
        diag = (wa2 == 0.) ? 1. : wa2;
        xnorm = fabs(diag * x);
        delta = factor * xnorm;
        if (delta == 0.) delta = factor;
      }
      qtf = (wa2 != 0.) ? jf / r00 : 0.0;
      gnorm = 0.;
      if (fnorm != 0. && wa2 != 0.) gnorm = fabs(r00 * (qtf / fnorm)) / wa2;
      if (gnorm <= 0.) {
        iteration++;
        if (iteration >= dc.max_iter) done = true;
        continue;
      }
      diag = fmax(diag, wa2);
      pstep = -lmpar_1d(r00, diag, qtf, delta, par);
      xn = x + pstep;
      pnorm = fabs(diag * pstep);
      if (iter == 1) delta = fmin(delta, pnorm);
      phase = 1;
      step_finished = false;
    }
  }
  if (lane == 0) {
    atomicAdd(&a.counters[6], (unsigned long long)nfev);
    atomicAdd(&a.counters[7], (unsigned long long)nexec);
    const int okx = !(x <= 0.001);
    const double inv = (r00 != 0.) ? (1. / r00) * (1. / r00) : 0.0;
    a.flag[k] = okx;
    a.res[3 * k] = x; a.res[3 * k + 1] = (dc.td_stdvar * dc.td_stdvar) * inv; a.res[3 * k + 2] = fnorm * fnorm;
  }
}

// --------------------------------------------------------------------------------------------
// Ordered compaction of solver results into DepthPoints (DepthProblemSolver.cpp:100-135) with
// optional pointCulling (:217-244) fused in; same thread-major order as seeds_order_kernel.
// --------------------------------------------------------------------------------------------
__device__ int block_excl_scan(int v, int* s_warp, int& total);

struct CullArgs { int enable; double var_thr, cost_thr, rmin, rmax; };

__device__ __forceinline__ int tm_index2(int v, int n, int NT) {
  int c = 0, start = 0;
  for (; c < NT; ++c) {
    const int members = (n > c) ? (n - c + NT - 1) / NT : 0;
    if (v < start + members) break;
    start += members;
  }
  return c + (v - start) * NT;
}
// Multi-block, no inter-block communication (same scheme as seeds_order_kernel, bm.cu): block b counts the kept seeds at the
// earlier virtual positions itself, scans its own 256 and writes its DepthPoints; the last block publishes the totals.
constexpr int kOrdBlockP = 256;
__global__ void __launch_bounds__(kOrdBlockP) points_order_kernel(DevConsts dc, const esvo_seed* __restrict__ seeds,
                                                                  const unsigned long long* n_ptr, int n_fixed,
                                                                  const int32_t* __restrict__ flag, const double* __restrict__ res,
                                                                  CullArgs cull, esvo_depth_point* out, unsigned long long* out_cnt,
                                                                  unsigned long long* counters) {
  __shared__ int s_warp[33];
  __shared__ int s_base, s_solved_pre;
  const int n = n_ptr ? (int)*n_ptr : n_fixed;
  const int NT = dc.NT;
  const int v0 = blockIdx.x * kOrdBlockP;
  if (v0 >= n) {
    if (blockIdx.x == 0 && threadIdx.x == 0) { counters[2] = 0; counters[3] = 0; if (out_cnt) *out_cnt = 0; }   // no seeds at all
    return;
  }
  auto keep = [&](int i) -> bool {
    if (!flag[i]) return false;
    if (!cull.enable) return true;
    const double rho = res[3 * i], var = res[3 * i + 1], cost = res[3 * i + 2];
    return var <= cull.var_thr && cost <= cull.cost_thr && rho > -1e-6 && rho >= cull.rmin && rho <= cull.rmax;
  };
  int pre = 0, pre_solved = 0;
  for (int v = threadIdx.x; v < v0; v += kOrdBlockP) { const int i = tm_index2(v, n, NT); pre += keep(i); pre_solved += flag[i] != 0; }
  int tot_pre, tot_solved_pre;
  block_excl_scan(pre, s_warp, tot_pre);
  block_excl_scan(pre_solved, s_warp, tot_solved_pre);
  if (threadIdx.x == 0) { s_base = tot_pre; s_solved_pre = tot_solved_pre; }
  const int v = v0 + threadIdx.x;
  const int i = v < n ? tm_index2(v, n, NT) : 0;
  const int kp = (v < n && keep(i)) ? 1 : 0;
  const int sv = (v < n && flag[i] != 0) ? 1 : 0;
  int total, total_solved;
  const int local = block_excl_scan(kp, s_warp, total);
  block_excl_scan(sv, s_warp, total_solved);
  if (kp) {
    const double rho = res[3 * i], var = res[3 * i + 1], cost = res[3 * i + 2];
    const esvo_seed& s = seeds[i];
    esvo_depth_point d;
    d.row = (int32_t)floor(s.x_left[1]); d.col = (int32_t)floor(s.x_left[0]);
    d.x[0] = s.x_left[0]; d.x[1] = s.x_left[1];
    cam2world_dev(dc, s.x_left[0], s.x_left[1], rho, d.p_cam);
    d.inv_depth = rho;
    if (dc.lsnorm == ESVO_LSNORM_L2) { d.variance = var < 1e-6 ? 1e-6 : var; d.scale2 = 0; d.nu = 0; }
    else { d.scale2 = var * (dc.td_nu - 2) / dc.td_nu; d.nu = dc.td_nu; d.variance = var; }
    d.residual = cost; d.age = 0;
#pragma unroll
    for (int q = 0; q < 16; ++q) d.T_world_cam[q] = s.T_world_virtual[q];
    out[s_base + local] = d;
  }
  if (v0 + kOrdBlockP >= n && threadIdx.x == 0) {
    counters[2] = (unsigned long long)(s_solved_pre + total_solved); counters[3] = (unsigned long long)(s_base + total);
    if (out_cnt) *out_cnt = (unsigned long long)(s_base + total);
  }
}

// pointCulling on an already ordered DepthPoint array (esvo_depth_cull): order-preserving compaction.
__global__ void __launch_bounds__(1024) cull_points_kernel(esvo_depth_point* pts, int n, CullArgs cull, esvo_depth_point* out,
                                                           unsigned long long* counters) {
  __shared__ int s_warp[33];
  int running = 0;
  for (int k0 = 0; k0 < n; k0 += blockDim.x) {
    const int i = k0 + threadIdx.x;
    int f = 0;
    esvo_depth_point d;
    if (i < n) {
      d = pts[i];
      f = (d.variance <= cull.var_thr && d.residual <= cull.cost_thr && d.inv_depth > -1e-6 && d.inv_depth >= cull.rmin &&
           d.inv_depth <= cull.rmax);
    }
    int total;
    const int pos = running + block_excl_scan(f, s_warp, total);
    if (f) out[pos] = d;
    running += total;
  }
  if (threadIdx.x == 0) counters[3] = (unsigned long long)running;
}

int lm_run(Ctx* c, const esvo_seed* d_seeds, size_t n_fixed) {
  const SlotBufs& f = c->slot();
  LmArgs a;
  a.seeds = d_seeds; a.n_ptr = n_fixed ? nullptr : (const unsigned long long*)(f.d_counters + 1);
  a.n_fixed = (int)n_fixed; a.tl = f.obs_ls; a.tr = f.obs_rs; std::memcpy(a.T_left_world, f.T_left_world_inv, sizeof(a.T_left_world));
  a.flag = f.lm_flag; a.res = f.lm_res; a.counters = (unsigned long long*)f.d_counters;
  const int upper = (int)(n_fixed ? n_fixed : f.n_ev);
  if (upper == 0) return ESVO_OK;
  // Tdist with up to 7 slots per lane: lm2_kernel at 20 seeds per SM.  On an H100 SXM (700 W limit, bench.py --no-parity
  // --no-extras --no-cpu-baseline) 20 beat 16 / 24 / 32 seeds per SM both as an isolated launch (0.62 vs 0.64 / 0.73 /
  // 0.82 ms) and in the 16-slot pipeline (0.237 vs 0.240 / 0.238 / 0.257 ms/step); see DESIGN.md §4.
  const bool td = c->dc.lsnorm == ESVO_LSNORM_TDIST;
  const bool s7 = c->dc.wx * c->dc.wy <= 7 * 16;
  if (td && s7) lm2_kernel<7, 20><<<upper, 32, 0, c->stream>>>(c->dc, a);
  else if (!s7) { if (td) lm_kernel<8, true><<<upper, 32, 0, c->stream>>>(c->dc, a); else lm_kernel<8, false><<<upper, 32, 0, c->stream>>>(c->dc, a); }
  else lm_kernel<7, false><<<upper, 32, 0, c->stream>>>(c->dc, a);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

// cull != 0: fuse pointCulling; out == null: the slot's d_pts.
int points_order_impl(Ctx* c, const esvo_seed* d_seeds, size_t n_fixed, int cull, double std_thr, double cost_thr,
                      double rmin, double rmax, esvo_depth_point* out, unsigned long long* out_cnt) {
  const SlotBufs& f = c->slot();
  CullArgs ca{cull, std_thr * std_thr, cost_thr, rmin, rmax};
  // the seed count lives on the device in the whole-frame path: the grid covers the event capacity, surplus blocks exit
  const int upper = (int)(n_fixed ? n_fixed : f.n_ev);
  points_order_kernel<<<std::max(1, div_up(upper, kOrdBlockP)), kOrdBlockP, 0, c->stream>>>(
      c->dc, d_seeds, n_fixed ? nullptr : (const unsigned long long*)(f.d_counters + 1), (int)n_fixed, f.lm_flag, f.lm_res, ca,
      out ? out : f.d_pts, out_cnt, (unsigned long long*)f.d_counters);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}
// in: d_pts[0..n) (device), out: the slot's d_pts, count in counters[3]
int cull_points(Ctx* c, esvo_depth_point* d_in, size_t n, double std_thr, double cost_thr, double rmin, double rmax) {
  const SlotBufs& f = c->slot();
  CullArgs ca{1, std_thr * std_thr, cost_thr, rmin, rmax};
  cull_points_kernel<<<1, kOrderThreads, 0, c->stream>>>(d_in, (int)n, ca, f.d_pts, (unsigned long long*)f.d_counters);
  c->launches += 1;
  ESVO_CUDA_TRY(c, cudaGetLastError());
  return ESVO_OK;
}

}  // namespace esvo
