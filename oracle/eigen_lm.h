// ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into or called from the product path.
//
// Restatement of the third-party numerical code the reference calls but does not vendor:
//   Eigen 3 (eigen_catkin "master", dependencies.yaml:22-25; README.md:71 "Eigen 3"):
//     unsupported/Eigen/NonLinearOptimization  LevenbergMarquardt::{minimizeInit,minimizeOneStep},
//     internal::{lmpar2, qrsolv, covar}; unsupported/Eigen/NumericalDiff (Forward);
//     Eigen/QR ColPivHouseholderQR (3.3 norm-downdating variant); Eigen/Jacobi 2x2 Givens.
//   These are ports of MINPACK lmder/lmpar/qrsolv/covar; the algorithm is restated from the
//   published MINPACK/Eigen sources.  Pinned in tests against scipy.optimize.leastsq (MINPACK
//   lmdif) iterates.
// Reference call sites: DepthProblemSolver.cpp:146-212 (n=1), RegProblemSolverLM.cpp:78-100,
// 150-176 (n=6).
#pragma once
#include <algorithm>
#include <cmath>
#include <functional>
#include <limits>
#include <vector>

namespace oracle {

struct ColPivQR {
  int m = 0, n = 0;
  std::vector<double> qr;     // column-major m x n, R in the upper triangle, essentials below
  std::vector<double> tau;    // n
  std::vector<int> perm;      // perm[j] = original column at position j
  double maxpivot = 0;
  int nonzero_pivots = 0;
  int downdate_recomputes = 0;   // trace only: columns whose norm the downdate re-computed instead of updating
  double& at(int i, int j) { return qr[(size_t)j * m + i]; }
  double at(int i, int j) const { return qr[(size_t)j * m + i]; }

  // Eigen/src/QR/ColPivHouseholderQR.h computeInPlace (3.3.x).
  void compute(const std::vector<double>& A, int m_, int n_) {
    m = m_; n = n_; qr = A;
    const int size = std::min(m, n);
    tau.assign(size, 0.0);
    std::vector<int> transp(n);
    std::vector<double> normsUpdated(n), normsDirect(n);
    for (int k = 0; k < n; ++k) {
      double s = 0;
      for (int i = 0; i < m; ++i) s += at(i, k) * at(i, k);
      normsDirect[k] = normsUpdated[k] = std::sqrt(s);
    }
    const double eps = std::numeric_limits<double>::epsilon();
    double mx = 0;
    for (int k = 0; k < n; ++k) mx = std::max(mx, normsUpdated[k]);
    const double threshold_helper = (mx * eps / m) * (mx * eps / m);
    const double norm_downdate_threshold = std::sqrt(eps);
    nonzero_pivots = size;
    maxpivot = 0;
    downdate_recomputes = 0;
    for (int k = 0; k < size; ++k) {
      int big = k;
      double bigv = normsUpdated[k];
      for (int j = k + 1; j < n; ++j)
        if (normsUpdated[j] > bigv) { bigv = normsUpdated[j]; big = j; }
      double big_sq = bigv * bigv;
      if (nonzero_pivots == size && big_sq < threshold_helper * (double)(m - k)) nonzero_pivots = k;
      transp[k] = big;
      if (k != big) {
        for (int i = 0; i < m; ++i) std::swap(at(i, k), at(i, big));
        std::swap(normsUpdated[k], normsUpdated[big]);
        std::swap(normsDirect[k], normsDirect[big]);
      }
      // makeHouseholderInPlace on col(k).tail(m-k)
      double c0 = at(k, k), tailSq = 0;
      for (int i = k + 1; i < m; ++i) tailSq += at(i, k) * at(i, k);
      double beta, t;
      const double tol = std::numeric_limits<double>::min();
      if (tailSq <= tol) {
        t = 0; beta = c0;
        for (int i = k + 1; i < m; ++i) at(i, k) = 0;
      } else {
        beta = std::sqrt(c0 * c0 + tailSq);
        if (c0 >= 0) beta = -beta;
        for (int i = k + 1; i < m; ++i) at(i, k) = at(i, k) / (c0 - beta);
        t = (beta - c0) / beta;
      }
      tau[k] = t;
      at(k, k) = beta;
      if (std::fabs(beta) > maxpivot) maxpivot = std::fabs(beta);
      // apply H_k to the trailing columns
      for (int j = k + 1; j < n; ++j) {
        if (m - k == 1) { at(k, j) *= (1 - t); continue; }
        if (t == 0) continue;
        double tmp = 0;
        for (int i = k + 1; i < m; ++i) tmp += at(i, k) * at(i, j);
        tmp += at(k, j);
        at(k, j) -= t * tmp;
        for (int i = k + 1; i < m; ++i) at(i, j) -= t * at(i, k) * tmp;
      }
      // norm downdate (LAPACK working note 176)
      for (int j = k + 1; j < n; ++j) {
        if (normsUpdated[j] != 0) {
          double temp = std::fabs(at(k, j)) / normsUpdated[j];
          temp = (1 + temp) * (1 - temp);
          temp = temp < 0 ? 0 : temp;
          double r = normsUpdated[j] / normsDirect[j];
          double temp2 = temp * r * r;
          if (temp2 <= norm_downdate_threshold) {
            double s = 0;
            for (int i = k + 1; i < m; ++i) s += at(i, j) * at(i, j);
            normsDirect[j] = std::sqrt(s);
            normsUpdated[j] = normsDirect[j];
            ++downdate_recomputes;
          } else {
            normsUpdated[j] *= std::sqrt(temp);
          }
        }
      }
    }
    perm.resize(n);
    for (int j = 0; j < n; ++j) perm[j] = j;
    for (int k = 0; k < size; ++k) std::swap(perm[k], perm[transp[k]]);
  }
  // rank() with the default threshold eps*diagonalSize
  int rank() const {
    const double thr = std::fabs(maxpivot) * std::numeric_limits<double>::epsilon() * std::min(m, n);
    int r = 0;
    for (int i = 0; i < nonzero_pivots; ++i) r += (std::fabs(at(i, i)) > thr);
    return r;
  }
  // v <- Q^T v  (householderQ().adjoint() applied on the left)
  void applyQt(std::vector<double>& v) const {
    const int size = std::min(m, n);
    for (int k = 0; k < size; ++k) {
      if (m - k == 1) { v[k] *= (1 - tau[k]); continue; }
      if (tau[k] == 0) continue;
      double tmp = 0;
      for (int i = k + 1; i < m; ++i) tmp += at(i, k) * v[i];
      tmp += v[k];
      v[k] -= tau[k] * tmp;
      for (int i = k + 1; i < m; ++i) v[i] -= tau[k] * at(i, k) * tmp;
    }
  }
};

static inline double vnorm(const double* v, int n) {
  double s = 0;
  for (int i = 0; i < n; ++i) s += v[i] * v[i];
  return std::sqrt(s);
}

// Eigen JacobiRotation::makeGivens(p, q) (real case)
static inline void make_givens(double p, double q, double& c, double& s) {
  if (q == 0) { c = p < 0 ? -1 : 1; s = 0; }
  else if (p == 0) { c = 0; s = q < 0 ? 1 : -1; }
  else if (std::fabs(p) > std::fabs(q)) {
    double t = q / p, u = std::sqrt(1 + t * t);
    if (p < 0) u = -u;
    c = 1 / u; s = -t * c;
  } else {
    double t = p / q, u = std::sqrt(1 + t * t);
    if (q < 0) u = -u;
    s = -1 / u; c = -t * s;
  }
}

// internal::qrsolv (s: n x n column-major copy of R's top block, modified in the lower triangle)
static inline void qrsolv(std::vector<double>& s, int n, const std::vector<int>& ipvt,
                          const std::vector<double>& diag, const std::vector<double>& qtb,
                          std::vector<double>& x, std::vector<double>& sdiag) {
  auto S = [&](int i, int j) -> double& { return s[(size_t)j * n + i]; };
  std::vector<double> wa(qtb.begin(), qtb.begin() + n);
  x.resize(n); sdiag.assign(n, 0.0);
  for (int j = 0; j < n; ++j) x[j] = S(j, j);
  for (int j = 0; j < n; ++j)
    for (int i = j + 1; i < n; ++i) S(i, j) = S(j, i);
  for (int j = 0; j < n; ++j) {
    int l = ipvt[j];
    if (diag[l] == 0.) break;
    for (int k = j; k < n; ++k) sdiag[k] = 0;
    sdiag[j] = diag[l];
    double qtbpj = 0.;
    for (int k = j; k < n; ++k) {
      double c, sn;
      make_givens(-S(k, k), sdiag[k], c, sn);
      S(k, k) = c * S(k, k) + sn * sdiag[k];
      double temp = c * wa[k] + sn * qtbpj;
      qtbpj = -sn * wa[k] + c * qtbpj;
      wa[k] = temp;
      for (int i = k + 1; i < n; ++i) {
        temp = c * S(i, k) + sn * sdiag[i];
        sdiag[i] = -sn * S(i, k) + c * sdiag[i];
        S(i, k) = temp;
      }
    }
  }
  int nsing = 0;
  for (nsing = 0; nsing < n && sdiag[nsing] != 0; nsing++) {}
  for (int j = nsing; j < n; ++j) wa[j] = 0;
  // solve (s.topLeft(nsing,nsing)^T as upper) z = wa: upper(i,j) = S(j,i) with diagonal S(i,i)
  for (int i = nsing - 1; i >= 0; --i) {
    double sum = wa[i];
    for (int j = i + 1; j < nsing; ++j) sum -= S(j, i) * wa[j];
    wa[i] = sum / S(i, i);
  }
  for (int j = 0; j < n; ++j) sdiag[j] = S(j, j);
  for (int j = 0; j < n; ++j) S(j, j) = x[j];
  for (int j = 0; j < n; ++j) x[ipvt[j]] = wa[j];
}

// internal::lmpar2.  n_iter (optional, trace only) receives the number of passes of the par
// iteration: 0 when the Gauss-Newton step already lies within 10 % of the trust region (par = 0).
static inline void lmpar2(const ColPivQR& qr, const std::vector<double>& diag,
                          const std::vector<double>& qtb, double delta, double& par,
                          std::vector<double>& x, int* n_iter = nullptr) {
  const double dwarf = std::numeric_limits<double>::min();
  const int n = qr.n;
  std::vector<double> wa1(qtb.begin(), qtb.begin() + n), wa2(n);
  const int rank = qr.rank();
  for (int j = rank; j < n; ++j) wa1[j] = 0;
  for (int i = rank - 1; i >= 0; --i) {  // R(0:rank,0:rank) upper solve
    double sum = wa1[i];
    for (int j = i + 1; j < rank; ++j) sum -= qr.at(i, j) * wa1[j];
    wa1[i] = sum / qr.at(i, i);
  }
  x.assign(n, 0.0);
  for (int j = 0; j < n; ++j) x[qr.perm[j]] = wa1[j];
  int iter = 0;
  for (int j = 0; j < n; ++j) wa2[j] = diag[j] * x[j];
  double dxnorm = vnorm(wa2.data(), n);
  double fp = dxnorm - delta;
  if (n_iter) *n_iter = 0;
  if (fp <= 0.1 * delta) { par = 0; return; }
  double parl = 0.;
  if (rank == n) {
    for (int j = 0; j < n; ++j) wa1[j] = diag[qr.perm[j]] * wa2[qr.perm[j]] / dxnorm;
    // solve R^T (lower) w = wa1
    for (int i = 0; i < n; ++i) {
      double sum = wa1[i];
      for (int j = 0; j < i; ++j) sum -= qr.at(j, i) * wa1[j];
      wa1[i] = sum / qr.at(i, i);
    }
    double temp = vnorm(wa1.data(), n);
    parl = fp / delta / temp / temp;
  }
  for (int j = 0; j < n; ++j) {
    double s = 0;
    for (int i = 0; i <= j; ++i) s += qr.at(i, j) * qtb[i];
    wa1[j] = s / diag[qr.perm[j]];
  }
  double gnorm = vnorm(wa1.data(), n);
  double paru = gnorm / delta;
  if (paru == 0.) paru = dwarf / std::min(delta, 0.1);
  par = std::max(par, parl);
  par = std::min(par, paru);
  if (par == 0.) par = gnorm / dxnorm;
  std::vector<double> s((size_t)n * n);
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < n; ++i) s[(size_t)j * n + i] = qr.at(i, j);
  std::vector<double> sdiag(n);
  while (true) {
    ++iter;
    if (par == 0.) par = std::max(dwarf, .001 * paru);
    double sp = std::sqrt(par);
    for (int j = 0; j < n; ++j) wa1[j] = sp * diag[j];
    qrsolv(s, n, qr.perm, wa1, qtb, x, sdiag);
    for (int j = 0; j < n; ++j) wa2[j] = diag[j] * x[j];
    dxnorm = vnorm(wa2.data(), n);
    double temp = fp;
    fp = dxnorm - delta;
    if (std::fabs(fp) <= 0.1 * delta || (parl == 0. && fp <= temp && temp < 0.) || iter == 10) break;
    for (int j = 0; j < n; ++j) wa1[j] = diag[qr.perm[j]] * (wa2[qr.perm[j]] / dxnorm);
    for (int j = 0; j < n; ++j) {
      wa1[j] /= sdiag[j];
      temp = wa1[j];
      for (int i = j + 1; i < n; ++i) wa1[i] -= s[(size_t)j * n + i] * temp;
    }
    temp = vnorm(wa1.data(), n);
    double parc = fp / delta / temp / temp;
    if (fp > 0.) parl = std::max(parl, par);
    if (fp < 0.) paru = std::min(paru, par);
    par = std::max(parl, par + parc);
  }
  if (iter == 0) par = 0.;
  if (n_iter) *n_iter = iter;
}

enum LMStatus {
  LM_NotStarted = -2, LM_Running = -1, LM_ImproperInputParameters = 0,
  LM_RelativeReductionTooSmall = 1, LM_RelativeErrorTooSmall = 2,
  LM_RelativeErrorAndReductionTooSmall = 3, LM_CosinusTooSmall = 4,
  LM_TooManyFunctionEvaluation = 5, LM_FtolTooSmall = 6, LM_XtolTooSmall = 7,
  LM_GtolTooSmall = 8, LM_UserAsked = 9
};

// Optional record of one minimizeOneStep (test infrastructure: recording changes no arithmetic).
struct LMStepTrace {
  struct Trial {
    std::vector<double> x;                       // the trial point x + p
    double fnorm1, actred, prered, ratio;
    double par, delta, xnorm;                    // after the trust-region update of this trial
    bool accepted;
    int lmpar_iter;                              // 0: lmpar returned early with par = 0
  };
  int rank = 0, nonzero_pivots = 0, downdate_recomputes = 0;
  double fnorm = 0, gnorm = 0;                   // at the start of the step
  std::vector<Trial> trials;
};

// f(x, fvec) -> <0 aborts;  df(x, fjac col-major m x n) -> number of f evaluations (numerical
// differentiation) or 0 (analytic).
struct LevenbergMarquardt {
  using Fn = std::function<int(const std::vector<double>&, std::vector<double>&)>;
  using DFn = std::function<int(const std::vector<double>&, std::vector<double>&)>;
  Fn f; DFn df; int m = 0, n = 0;
  // parameters (resetParameters defaults)
  double factor = 100., ftol, xtol, gtol = 0., epsfcn = 0.;
  int maxfev = 400;
  // state
  std::vector<double> fvec, fjac, diag, qtf, wa1, wa2, wa3, wa4;
  ColPivQR qrfac;
  int nfev = 0, njev = 0, iter = 0;
  double fnorm = 0, gnorm = 0, par = 0, xnorm = 0, delta = 0;
  LMStepTrace* trace = nullptr;   // filled by minimizeOneStep when set

  LevenbergMarquardt() { ftol = xtol = std::sqrt(std::numeric_limits<double>::epsilon()); }

  LMStatus minimizeInit(std::vector<double>& x, int m_values) {
    n = (int)x.size(); m = m_values;
    wa1.assign(n, 0); wa2.assign(n, 0); wa3.assign(n, 0); wa4.assign(m, 0);
    fvec.assign(m, 0); fjac.assign((size_t)m * n, 0); diag.assign(n, 0); qtf.assign(n, 0);
    nfev = 0; njev = 0;
    if (n <= 0 || m < n || ftol < 0. || xtol < 0. || gtol < 0. || maxfev <= 0 || factor <= 0.)
      return LM_ImproperInputParameters;
    nfev = 1;
    if (f(x, fvec) < 0) return LM_UserAsked;
    fnorm = vnorm(fvec.data(), m);
    par = 0.; iter = 1;
    return LM_NotStarted;
  }

  LMStatus minimizeOneStep(std::vector<double>& x) {
    const double eps = std::numeric_limits<double>::epsilon();
    int df_ret = df(x, fjac);
    if (df_ret < 0) return LM_UserAsked;
    if (df_ret > 0) nfev += df_ret; else njev++;
    for (int j = 0; j < n; ++j) wa2[j] = vnorm(&fjac[(size_t)j * m], m);
    qrfac.compute(fjac, m, n);
    fjac = qrfac.qr;
    const std::vector<int>& perm = qrfac.perm;
    if (trace) {
      *trace = LMStepTrace();
      trace->rank = qrfac.rank(); trace->nonzero_pivots = qrfac.nonzero_pivots;
      trace->downdate_recomputes = qrfac.downdate_recomputes; trace->fnorm = fnorm;
    }
    if (iter == 1) {
      for (int j = 0; j < n; ++j) diag[j] = (wa2[j] == 0.) ? 1. : wa2[j];
      double s = 0;
      for (int j = 0; j < n; ++j) s += (diag[j] * x[j]) * (diag[j] * x[j]);
      xnorm = std::sqrt(s);
      delta = factor * xnorm;
      if (delta == 0.) delta = factor;
    }
    wa4 = fvec;
    qrfac.applyQt(wa4);
    for (int j = 0; j < n; ++j) qtf[j] = wa4[j];
    gnorm = 0.;
    if (fnorm != 0.)
      for (int j = 0; j < n; ++j)
        if (wa2[perm[j]] != 0.) {
          double s = 0;
          for (int i = 0; i <= j; ++i) s += qrfac.at(i, j) * (qtf[i] / fnorm);
          gnorm = std::max(gnorm, std::fabs(s / wa2[perm[j]]));
        }
    if (trace) trace->gnorm = gnorm;
    if (gnorm <= gtol) return LM_CosinusTooSmall;
    for (int j = 0; j < n; ++j) diag[j] = std::max(diag[j], wa2[j]);
    double ratio;
    do {
      int lmpar_iter = 0;
      lmpar2(qrfac, diag, qtf, delta, par, wa1, &lmpar_iter);
      for (int j = 0; j < n; ++j) { wa1[j] = -wa1[j]; wa2[j] = x[j] + wa1[j]; }
      double s = 0;
      for (int j = 0; j < n; ++j) s += (diag[j] * wa1[j]) * (diag[j] * wa1[j]);
      double pnorm = std::sqrt(s);
      if (iter == 1) delta = std::min(delta, pnorm);
      if (f(wa2, wa4) < 0) return LM_UserAsked;
      ++nfev;
      double fnorm1 = vnorm(wa4.data(), m);
      double actred = -1.;
      if (.1 * fnorm1 < fnorm) actred = 1. - (fnorm1 / fnorm) * (fnorm1 / fnorm);
      // wa3 = R * (P^-1 wa1)
      for (int i = 0; i < n; ++i) {
        double t = 0;
        for (int j = i; j < n; ++j) t += qrfac.at(i, j) * wa1[perm[j]];
        wa3[i] = t;
      }
      double t1 = vnorm(wa3.data(), n) / fnorm; double temp1 = t1 * t1;
      double t2 = std::sqrt(par) * pnorm / fnorm; double temp2 = t2 * t2;
      double prered = temp1 + temp2 / .5;
      double dirder = -(temp1 + temp2);
      ratio = 0.;
      if (prered != 0.) ratio = actred / prered;
      if (ratio <= .25) {
        double temp = 0;
        if (actred >= 0.) temp = .5;
        if (actred < 0.) temp = .5 * dirder / (dirder + .5 * actred);
        if (.1 * fnorm1 >= fnorm || temp < .1) temp = .1;
        delta = temp * std::min(delta, pnorm / .1);
        par /= temp;
      } else if (!(par != 0. && ratio < .75)) {
        delta = pnorm / .5;
        par = .5 * par;
      }
      if (ratio >= 1e-4) {
        x = wa2;
        double s2 = 0;
        for (int j = 0; j < n; ++j) { wa2[j] = diag[j] * x[j]; s2 += wa2[j] * wa2[j]; }
        fvec = wa4;
        xnorm = std::sqrt(s2);
        fnorm = fnorm1;
        ++iter;
      }
      if (trace)
        trace->trials.push_back({ratio >= 1e-4 ? x : wa2, fnorm1, actred, prered, ratio, par, delta, xnorm,
                                 ratio >= 1e-4, lmpar_iter});
      if (std::fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1. && delta <= xtol * xnorm)
        return LM_RelativeErrorAndReductionTooSmall;
      if (std::fabs(actred) <= ftol && prered <= ftol && .5 * ratio <= 1.)
        return LM_RelativeReductionTooSmall;
      if (delta <= xtol * xnorm) return LM_RelativeErrorTooSmall;
      if (nfev >= maxfev) return LM_TooManyFunctionEvaluation;
      if (std::fabs(actred) <= eps && prered <= eps && .5 * ratio <= 1.) return LM_FtolTooSmall;
      if (delta <= eps * xnorm) return LM_XtolTooSmall;
      if (gnorm <= eps) return LM_GtolTooSmall;
    } while (ratio < 1e-4);
    return LM_Running;
  }
};

// Eigen::NumericalDiff<F, Forward>::df : re-evaluates f(x), then one eval per column,
// h = sqrt(max(epsfcn, eps)) * |x_j| (or that constant if x_j == 0).  Returns n+1.
static inline int numerical_diff_forward(const LevenbergMarquardt::Fn& f, const std::vector<double>& x_,
                                         std::vector<double>& jac, int m, double epsfcn = 0.) {
  const int n = (int)x_.size();
  const double eps = std::sqrt(std::max(epsfcn, std::numeric_limits<double>::epsilon()));
  std::vector<double> x = x_, val1(m), val2(m);
  int nfev = 0;
  f(x, val1); nfev++;
  jac.assign((size_t)m * n, 0.0);
  for (int j = 0; j < n; ++j) {
    double h = eps * std::fabs(x[j]);
    if (h == 0.) h = eps;
    x[j] += h;
    f(x, val2); nfev++;
    x[j] = x_[j];
    for (int i = 0; i < m; ++i) jac[(size_t)j * m + i] = (val2[i] - val1[i]) / h;
  }
  return nfev;
}

// internal::covar specialised the way the reference uses it: returns element (0,0) of the
// covariance matrix after covar(lm.fjac, perm) (DepthProblemSolver.cpp:199).  General n.
static inline void covar(std::vector<double>& r, int m, int n, const std::vector<int>& ipvt) {
  auto R = [&](int i, int j) -> double& { return r[(size_t)j * m + i]; };
  const double tol = std::sqrt(std::numeric_limits<double>::epsilon());
  const double tolr = tol * std::fabs(R(0, 0));
  std::vector<double> wa(n);
  int l = -1;
  for (int k = 0; k < n; ++k)
    if (std::fabs(R(k, k)) > tolr) {
      R(k, k) = 1. / R(k, k);
      for (int j = 0; j <= k - 1; ++j) {
        double temp = R(k, k) * R(j, k);
        R(j, k) = 0.;
        for (int i = 0; i <= j; ++i) R(i, k) -= R(i, j) * temp;
      }
      l = k;
    }
  for (int k = 0; k <= l; ++k) {
    for (int j = 0; j <= k - 1; ++j) {
      double t = R(j, k);
      for (int i = 0; i <= j; ++i) R(i, j) += R(i, k) * t;
    }
    double t = R(k, k);
    for (int i = 0; i <= k; ++i) R(i, k) *= t;
  }
  for (int j = 0; j < n; ++j) {
    int jj = ipvt[j];
    bool sing = j > l;
    for (int i = 0; i <= j; ++i) {
      if (sing) R(i, j) = 0.;
      int ii = ipvt[i];
      if (ii > jj) R(ii, jj) = R(i, j);
      if (ii < jj) R(jj, ii) = R(i, j);
    }
    wa[jj] = R(j, j);
  }
  for (int j = 0; j < n; ++j) {
    for (int i = 0; i < j; ++i) R(i, j) = R(j, i);
    R(j, j) = wa[j];
  }
}

}  // namespace oracle
