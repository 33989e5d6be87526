// guided_oracle.cpp — CPU restatement of guided matching (DESIGN §3.9): geometry_aware::GuidedMatching
// (robust_estimation/guided_matching.hpp:28-68, 73-113, 178-227) with EpipolarDistanceError
// (multiview/solver_fundamental_kernel.cpp:157-166) or AsymmetricError (multiview/solver_homography_kernel.hpp:59-63)
// over flat arrays.  Compiled with -ffp-contract=off: every operation is rounded as the reference rounds it, including
// the fused multiply-adds the reference's x86-64-v3 build forms in M [x; 1] (EpipolarDistanceError::Error in
// solver_fundamental_kernel.cpp, Eigen's homogeneous product for AsymmetricError), written out with std::fma.
// Test infrastructure only.
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdint>

namespace {

// model 0: EpipolarDistanceError, 1: AsymmetricError; M row-major
inline double error(int model, const double *M, double x, double y, double u, double v) {
  if (model == 0) {
    const double p0 = std::fma(M[1], y, M[0] * x) + M[2], p1 = std::fma(M[4], y, M[3] * x) + M[5], p2 = std::fma(M[7], y, M[6] * x) + M[8];
    const double dt = p0 * u + p1 * v + p2;
    return dt * dt / (p0 * p0 + p1 * p1);
  }
  const double p0 = std::fma(M[0], x, M[1] * y) + M[2], p1 = std::fma(M[3], x, M[4] * y) + M[5], p2 = std::fma(M[6], x, M[7] * y) + M[8];
  const double dx = u - p0 / p2, dy = v - p1 / p2;
  return dx * dx + dy * dy;
}

// matching::L2<uint8_t> (matching/metric.hpp:55-93)
inline int l2(const uint8_t *a, const uint8_t *b) {
  int s = 0;
  for (int k = 0; k < 128; ++k) { const int d = int(a[k]) - int(b[k]); s += d * d; }
  return s;
}

}  // namespace

extern "C" {

// errors of n (x_i, y_i) pairs against one model (validation of the boundary cases)
void oracle_guided_errors(int model, const double *M, const double *xI, const double *xJ, uint32_t n, double *err) {
  for (uint32_t k = 0; k < n; ++k) err[k] = error(model, M, xI[2 * k], xI[2 * k + 1], xJ[2 * k], xJ[2 * k + 1]);
}

// One pair.  ratio >= 0: the descriptor variant (distanceRatio<double>, isValid(ratio)); ratio < 0: the descriptor-free
// variant (lowest j of minimal error < thr).  out_ij[nI][2]: (i, j) in ascending i; returns the number of matches.
uint32_t oracle_guided(int model, const double *xI, uint32_t nI, const uint8_t *dI, const double *xJ, uint32_t nJ,
                       const uint8_t *dJ, const double *M, double thr, double ratio, uint32_t *out_ij) {
  uint32_t n = 0;
  for (uint32_t i = 0; i < nI; ++i) {
    if (ratio >= 0) {
      double bd = DBL_MAX, sbd = DBL_MAX; uint32_t idx = 0;
      for (uint32_t j = 0; j < nJ; ++j) {
        const double e = error(model, M, xI[2 * i], xI[2 * i + 1], xJ[2 * j], xJ[2 * j + 1]);
        if (!(e < thr)) continue;
        const double d = l2(dI + 128 * (size_t)i, dJ + 128 * (size_t)j);
        if (d < bd) { idx = j; sbd = bd; bd = d; } else if (d < sbd) sbd = d;
      }
      if (sbd != DBL_MAX && bd < ratio * sbd) { out_ij[2 * n] = i; out_ij[2 * n + 1] = idx; ++n; }
    } else {
      double mn = DBL_MAX; uint32_t idx = 0;
      for (uint32_t j = 0; j < nJ; ++j) {
        const double e = error(model, M, xI[2 * i], xI[2 * i + 1], xJ[2 * j], xJ[2 * j + 1]);
        if (e < thr && e < mn) { mn = e; idx = j; }
      }
      if (mn < thr) { out_ij[2 * n] = i; out_ij[2 * n + 1] = idx; ++n; }
    }
  }
  return n;
}

}  // extern "C"
