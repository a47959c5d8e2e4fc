// ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into or called from the product path.
//
// CPU restatement of the tracking residual/Jacobian and its LM driver:
//   esvo_core/src/core/RegProblemLM.cpp, RegProblemSolverLM.cpp, tools/cayley.cpp.
#pragma once
#include "o_mapping.h"

namespace oracle {

// glibc rand()/srand() (TYPE_3 additive feedback generator, r[i] = r[i-3] + r[i-31]), restated
// so that each context owns its own stream; the reference calls the process-global rand()
// without ever seeding it (RegProblemLM.cpp:49) == srand(1).  Pinned against libc in tests.
struct GlibcRand {
  int32_t r[34];
  uint32_t hist[31];
  int pos = 0;
  GlibcRand() { seed(1); }
  void seed(unsigned s) {
    if (s == 0) s = 1;
    std::vector<uint32_t> v(344);
    int32_t word = (int32_t)s;
    v[0] = (uint32_t)word;
    for (int i = 1; i < 31; ++i) {
      long hi = word / 127773, lo = word % 127773;
      word = (int32_t)(16807 * lo - 2836 * hi);
      if (word < 0) word += 2147483647;
      v[i] = (uint32_t)word;
    }
    for (int i = 31; i < 34; ++i) v[i] = v[i - 31];
    for (int i = 34; i < 344; ++i) v[i] = v[i - 31] + v[i - 3];
    for (int i = 0; i < 31; ++i) hist[i] = v[344 - 31 + i];
    pos = 0;
  }
  int next() {
    // hist holds the last 31 outputs in a ring; new = o[k-31] + o[k-3]
    uint32_t a = hist[pos % 31];            // k-31
    uint32_t b = hist[(pos + 28) % 31];     // k-3
    uint32_t n = a + b;
    hist[pos % 31] = n;
    pos = (pos + 1) % 31;
    return (int)(n >> 1);
  }
};

// tools::cayley2rot (cayley.cpp:4-21)
static inline void cayley2rot(const double c[3], double R[9]) {
  double scale = 1 + c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
  R[0] = 1 + c[0] * c[0] - c[1] * c[1] - c[2] * c[2];
  R[1] = 2 * (c[0] * c[1] - c[2]);
  R[2] = 2 * (c[0] * c[2] + c[1]);
  R[3] = 2 * (c[0] * c[1] + c[2]);
  R[4] = 1 - c[0] * c[0] + c[1] * c[1] - c[2] * c[2];
  R[5] = 2 * (c[1] * c[2] - c[0]);
  R[6] = 2 * (c[0] * c[2] - c[1]);
  R[7] = 2 * (c[1] * c[2] + c[0]);
  R[8] = 1 - c[0] * c[0] - c[1] * c[1] + c[2] * c[2];
  for (int i = 0; i < 9; ++i) R[i] = (1 / scale) * R[i];
}

// svd.matrixU() * svd.matrixV().transpose() of a 3x3 (JacobiSVD, RegProblemLM.cpp:336-337,
// 357-358) = the orthogonal polar factor M (M^T M)^{-1/2}, computed with a cyclic Jacobi
// eigen-decomposition of M^T M.
static inline void polar_orthonormalize(const double M[9], double Q[9]) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += M[k * 3 + i] * M[k * 3 + j];
      A[i * 3 + j] = s;
    }
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double apq = A[p * 3 + q];
        if (apq == 0) continue;
        double theta = (A[q * 3 + q] - A[p * 3 + p]) / (2 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
        double c = 1 / std::sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 3; ++k) {  // A <- A J
          double akp = A[k * 3 + p], akq = A[k * 3 + q];
          A[k * 3 + p] = c * akp - s * akq; A[k * 3 + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {  // A <- J^T A
          double apk = A[p * 3 + k], aqk = A[q * 3 + k];
          A[p * 3 + k] = c * apk - s * aqk; A[q * 3 + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
          V[k * 3 + p] = c * vkp - s * vkq; V[k * 3 + q] = s * vkp + c * vkq;
        }
      }
  }
  double isq[3] = {1 / std::sqrt(A[0]), 1 / std::sqrt(A[4]), 1 / std::sqrt(A[8])};
  double S[9];  // V diag(isq) V^T
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += V[i * 3 + k] * isq[k] * V[j * 3 + k];
      S[i * 3 + j] = s;
    }
  mat3_mul(M, S, Q);
}
static inline double det3(const double* A) {
  return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

struct RegProblem {
  const CameraSystem* cs = nullptr;
  esvo_params prm;
  TsObs* obs = nullptr;
  Mat4 T_world_ref, T_world_left;
  double R_[9], t_[3];
  double J_G_0[72];  // 12 x 6 row-major
  std::vector<double> ResItems;      // 3 per point (p in ref frame)
  std::vector<double> Sampled;       // current batch
  size_t numPoints = 0, numBatches = 1;
  GlibcRand rng;
  uint64_t n_evals = 0;
  // Trace of the last solve (test infrastructure), per outer iteration: TRACE_HEAD doubles {batch offset, m, status,
  // nfev, rank, nonzero_pivots, norm-downdate recomputes, number of trials, fnorm, gnorm, R_[9], t_[3] (the state the
  // iteration starts from)}, then per trial
  // TRACE_TRIAL doubles {x[6], fnorm1, actred, prered, ratio, par, delta, xnorm, accepted, lmpar iterations}.
  static constexpr int TRACE_HEAD = 22, TRACE_TRIAL = 15;
  std::vector<double> trace;

  // computeJ_G at x = 0 (RegProblemLM.cpp:271-320): only J_G_0_ is ever used (:21).
  void init() {
    std::memset(J_G_0, 0, sizeof(J_G_0));
    auto J = [&](int r, int c) -> double& { return J_G_0[r * 6 + c]; };
    // A1 = [[0,0,0],[0,0,2],[0,-2,0]], A2 = [[0,0,-2],[0,0,0],[2,0,0]], A3 = [[0,2,0],[-2,0,0],[0,0,0]]
    J(1, 2) = 2; J(2, 1) = -2;
    J(3, 2) = -2; J(5, 0) = 2;
    J(6, 1) = 2; J(7, 0) = -2;
    J(9, 3) = 1; J(10, 4) = 1; J(11, 5) = 1;
  }
  // setProblem (:24-68).  ref_xyz (n x 3 float, world frame) is permuted in place.
  void setProblem(float* ref_xyz, size_t n, const Mat4& Twr, const Mat4& Twc, TsObs* cur, bool bComputeGrad) {
    T_world_ref = Twr; T_world_left = Twc; obs = cur;
    double inv[16];
    inverse4(T_world_ref.m, inv);
    Mat4 T_ref_left = mul(Mat4::from(inv), T_world_left);
    for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R_[i * 3 + j] = T_ref_left(i, j); t_[i] = T_ref_left(i, 3); }
    numPoints = std::min(n, (size_t)prm.trk_max_registration_points);
    ResItems.assign(3 * numPoints, 0.0);
    for (size_t i = 0; i < numPoints; ++i) {
      size_t j = i + (size_t)rng.next() % (n - i);
      for (int k = 0; k < 3; ++k) std::swap(ref_xyz[3 * i + k], ref_xyz[3 * j + k]);
      double pt[3] = {(double)ref_xyz[3 * i], (double)ref_xyz[3 * i + 1], (double)ref_xyz[3 * i + 2]};
      double d[3] = {pt[0] - T_world_ref(0, 3), pt[1] - T_world_ref(1, 3), pt[2] - T_world_ref(2, 3)};
      for (int r = 0; r < 3; ++r)  // R_world_ref^T * d
        ResItems[3 * i + r] = T_world_ref(0, r) * d[0] + T_world_ref(1, r) * d[1] + T_world_ref(2, r) * d[2];
    }
    numBatches = std::max(numPoints / (size_t)prm.trk_batch_size, (size_t)1);
    obs->getTimeSurfaceNegative(prm.trk_kernel_size);
    if (bComputeGrad) obs->computeTsNegativeGrad();
  }
  // setStochasticSampling (:70-89)
  void setStochasticSampling(size_t offset, size_t N) {
    Sampled.clear();
    size_t total = ResItems.size() / 3;
    for (size_t i = 0; i < N; ++i) {
      if (offset + i >= total) break;
      for (int k = 0; k < 3; ++k) Sampled.push_back(ResItems[3 * (offset + i) + k]);
    }
    numPoints = Sampled.size() / 3;
  }
  // isValidPatch + reprojection (:380-416), patch 1x1
  bool reprojection(const double p[3], const double T[12], double x1[2]) const {
    double pl[3];
    for (int i = 0; i < 3; ++i) pl[i] = T[i * 4] * p[0] + T[i * 4 + 1] * p[1] + T[i * 4 + 2] * p[2] + T[i * 4 + 3];
    cs->left.world2Cam(pl, x1);
    const int W = cs->left.W, H = cs->left.H;
    if (x1[0] < 0 || x1[0] > W - 1 || x1[1] < 0 || x1[1] > H - 1) return false;
    if (cs->left.mask[(size_t)((long)x1[1]) * W + (size_t)((long)x1[0])] < 125) return false;
    return true;
  }
  // getWarpingTransformation (:322-346)
  int getWarpingTransformation(double T[12], const double* x) const {
    double dR[9], dRt[9], Rt[9], newR[9], Rcr[9];
    cayley2rot(x, dR);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { dRt[i * 3 + j] = dR[j * 3 + i]; Rt[i * 3 + j] = R_[j * 3 + i]; }
    mat3_mul(Rt, dRt, newR);
    polar_orthonormalize(newR, Rcr);
    if (det3(Rcr) < 0.0) return -1;
    double v[3];
    for (int i = 0; i < 3; ++i) v[i] = x[3 + i] + dR[i * 3] * t_[0] + dR[i * 3 + 1] * t_[1] + dR[i * 3 + 2] * t_[2];
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) T[i * 4 + j] = Rcr[i * 3 + j];
      T[i * 4 + 3] = -(Rcr[i * 3] * v[0] + Rcr[i * 3 + 1] * v[1] + Rcr[i * 3 + 2] * v[2]);
    }
    return 0;
  }
  // operator() + thread (:91-176)
  int residuals(const std::vector<double>& x, std::vector<double>& fvec) {
    n_evals++;
    double T[12];
    if (getWarpingTransformation(T, x.data()) < 0) return -1;
    for (size_t i = 0; i < numPoints; ++i) {
      double x1[2], r;
      if (!reprojection(&Sampled[3 * i], T, x1)) r = 255.0;
      else {
        double tau;
        if (patchInterpolation(obs->TS_negative_left.data(), obs->W, obs->H, x1, 1, 1, &tau)) r = tau;
        else r = 255.0;
      }
      if (prm.trk_lsnorm == ESVO_TRK_LSNORM_HUBER) {
        double w = 1.0;
        if (r > prm.trk_huber_threshold) w = prm.trk_huber_threshold / r;
        fvec[i] = std::sqrt(w) * r;
      } else fvec[i] = r;
    }
    return 0;
  }
  // df (:178-269), evaluated at x = 0 only; fjac column-major m x 6
  int jacobian(const std::vector<double>& x, std::vector<double>& fjac) {
    for (double v : x) if (v != 0) return -1;
    const size_t m = numPoints;
    fjac.assign(m * 6, 0.0);
    const double* P = cs->left.P;
    double Jc[6];  // 3x2 = R_^T * diag(1/P11, 1/P22, 0)[3x2]
    for (int i = 0; i < 3; ++i) { Jc[i * 2 + 0] = R_[0 * 3 + i] * (1.0 / P[0]); Jc[i * 2 + 1] = R_[1 * 3 + i] * (1.0 / P[5]); }
    double T[12];
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) T[i * 4 + j] = R_[j * 3 + i];
      T[i * 4 + 3] = -(R_[0 * 3 + i] * t_[0] + R_[1 * 3 + i] * t_[1] + R_[2 * 3 + i] * t_[2]);
    }
    const double P11 = P[0], P12 = P[1], P14 = P[3], P21 = P[4], P22 = P[5], P24 = P[7];
    for (size_t i = 0; i < m; ++i) {
      const double* p = &Sampled[3 * i];
      double x1[2], row12[12] = {0};
      if (reprojection(p, T, x1)) {
        double gx = 0, gy = 0;
        bool ok = patchInterpolation(obs->dTS_negative_du_left.data(), obs->W, obs->H, x1, 1, 1, &gx) &&
                  patchInterpolation(obs->dTS_negative_dv_left.data(), obs->W, obs->H, x1, 1, 1, &gy);
        if (ok) {  // (the reference reads an empty matrix here when interpolation fails: UB; zero row)
          double g[2] = {gx / 8, gy / 8};
          double dPi[6] = {P[0] / p[2], P[1] / p[2], 0, P[4] / p[2], P[5] / p[2], 0};
          const double z2 = p[2] * p[2];
          dPi[2] = -(P11 * p[0] + P12 * p[1] + P14) / z2;
          dPi[5] = -(P21 * p[0] + P22 * p[1] + P24) / z2;
          // ((((g^T dPi) Jc) dPi) dT_dG) * z   -- left-to-right like the Eigen expression
          double a[3], b[2], c[3];
          for (int k = 0; k < 3; ++k) a[k] = g[0] * dPi[k] + g[1] * dPi[3 + k];
          for (int k = 0; k < 2; ++k) b[k] = a[0] * Jc[k] + a[1] * Jc[2 + k] + a[2] * Jc[4 + k];
          for (int k = 0; k < 3; ++k) c[k] = b[0] * dPi[k] + b[1] * dPi[3 + k];
          for (int blk = 0; blk < 4; ++blk) {
            double s = blk < 3 ? p[blk] : 1.0;
            for (int k = 0; k < 3; ++k) row12[blk * 3 + k] = (c[k] * s) * p[2];
          }
        }
      }
      for (int j = 0; j < 6; ++j) {
        double s = 0;
        for (int k = 0; k < 12; ++k) s += row12[k] * J_G_0[k * 6 + j];
        fjac[(size_t)j * m + i] = -s;
      }
    }
    return 0;
  }
  // addMotionUpdate (:348-360)
  void addMotionUpdate(const double* dx) {
    double dR[9], newR[9], Rn[9];
    cayley2rot(dx, dR);
    mat3_mul(dR, R_, newR);
    polar_orthonormalize(newR, Rn);
    double tn[3];
    for (int i = 0; i < 3; ++i) tn[i] = dx[3 + i] + dR[i * 3] * t_[0] + dR[i * 3 + 1] * t_[1] + dR[i * 3 + 2] * t_[2];
    std::memcpy(R_, Rn, sizeof(R_)); std::memcpy(t_, tn, sizeof(t_));
  }
  // setPose (:362-372)
  void setPose() {
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += T_world_ref(i, k) * R_[k * 3 + j];
        T_world_left(i, j) = s;
      }
      T_world_left(i, 3) = T_world_ref(i, 0) * t_[0] + T_world_ref(i, 1) * t_[1] + T_world_ref(i, 2) * t_[2] + T_world_ref(i, 3);
    }
  }
  // RegProblemSolverLM::solve_analytical / solve_numerical (RegProblemSolverLM.cpp:76-217)
  int solve(bool analytical, esvo_lm_stats* st) {
    LevenbergMarquardt lm;
    lm.f = [&](const std::vector<double>& x, std::vector<double>& fv) { return residuals(x, fv); };
    if (analytical) lm.df = [&](const std::vector<double>& x, std::vector<double>& J) { return jacobian(x, J); };
    else lm.df = [&](const std::vector<double>& x, std::vector<double>& J) { return numerical_diff_forward(lm.f, x, J, (int)numPoints); };
    lm.ftol = 1e-3; lm.xtol = 1e-3; lm.maxfev = prm.trk_max_iteration * 8;
    size_t iteration = 0, nfev = 0;
    LMStepTrace step;
    lm.trace = &step;
    trace.clear();
    while (true) {
      if (iteration >= (size_t)prm.trk_max_iteration) break;
      const size_t offset = (iteration % numBatches) * prm.trk_batch_size;
      setStochasticSampling(offset, prm.trk_batch_size);
      std::vector<double> x(6, 0.0);
      double R0[9], t0[3];
      std::memcpy(R0, R_, sizeof(R0)); std::memcpy(t0, t_, sizeof(t0));
      if (lm.minimizeInit(x, (int)numPoints) == LM_ImproperInputParameters) return -1;
      LMStatus status = lm.minimizeOneStep(x);
      const double head[10] = {(double)offset, (double)numPoints, (double)status, (double)lm.nfev, (double)step.rank,
                               (double)step.nonzero_pivots, (double)step.downdate_recomputes, (double)step.trials.size(),
                               step.fnorm, step.gnorm};
      trace.insert(trace.end(), head, head + 10);
      trace.insert(trace.end(), R0, R0 + 9);
      trace.insert(trace.end(), t0, t0 + 3);
      for (const auto& t : step.trials) {
        trace.insert(trace.end(), t.x.begin(), t.x.end());
        const double rec[TRACE_TRIAL - 6] = {t.fnorm1, t.actred, t.prered, t.ratio, t.par, t.delta, t.xnorm,
                                             (double)t.accepted, (double)t.lmpar_iter};
        trace.insert(trace.end(), rec, rec + TRACE_TRIAL - 6);
      }
      addMotionUpdate(x.data());
      iteration++;
      nfev += lm.nfev;
      if (status == 2 || status == 3) break;
    }
    setPose();
    if (st) { st->n_points = (int64_t)numPoints; st->nfev = (int64_t)nfev; st->n_iter = (int64_t)iteration; }
    return 0;
  }
};

}  // namespace oracle
