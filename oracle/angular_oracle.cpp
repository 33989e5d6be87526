// angular_oracle.cpp — CPU restatement of the angular essential-matrix geometric filters that openMVG_main_GeometricFilter
// runs with `-g a` (eight-point) and `-g u` (upright three-point) (DESIGN §3.10).
//
// TEST INFRASTRUCTURE ONLY.  Built as its own library (oracle/_build/liboracle_angular.so, oracle/angular.mk); it
// includes acransac_oracle.cpp for the parts the F/H filter already restates: MT19937 + Lemire, the two UniformSample
// variants, the 9x9 Jacobi, the NFA tables and the quantified NFA.
//
// Parity status: PINNED by tests/test_oracle_geom_angular.py against oracle/_ref/libref_geom_angular.so (the reference's
// own EightPointRelativePoseSolver, ThreePointUprightRelativePoseSolver, AngularError, ACRANSAC +
// ACKernelAdaptor_AngularRadianError and RelativePoseFromEssential): solver outputs equal up to sign, AngularError bit for
// bit, identical cheirality counts, identical inlier lists before and after the cheirality step.
//
// Reference lines restated ($OPENMVG/src/openMVG):
//   matching_image_collection/E_ACRobust_Angular.hpp:52-160                 Robust_estimation (kernel, pose, keep rule)
//   robust_estimation/robust_estimator_ACRansacKernelAdaptator.hpp:465-539  ACKernelAdaptor_AngularRadianError
//   robust_estimation/robust_estimator_ACRansacKernelAdaptator.hpp:86-100   RADIAN_ANGLE: logalpha0 = log10(1/2), multError = 1/4
//   multiview/solver_essential_eight_point.cpp:15-60                        EightPointRelativePoseSolver, AngularError
//   multiview/solver_essential_three_point.cpp:86-114                       ThreePointUprightRelativePoseSolver
//   multiview/motion_from_essential.cpp:20-95                               RelativePoseFromEssential
//   multiview/essential.cpp:79-113                                          MotionFromEssential
//   multiview/triangulation.cpp:75-89,179-216                               AbsoluteToRelative, TriangulateIDWMidpoint
//   numeric/numeric.h:123-126                                               D2R
// The linear algebra the reference takes from Eigen is restated from the published algorithms instead:
//   SelfAdjointEigenSolver<9x9 | 4x4> -> cyclic Jacobi (the smallest eigenvector, up to sign; AngularError is sign-blind);
//   JacobiSVD<3x3> of E               -> Jacobi eigenvectors of E'E, u_i = E v_i / |E v_i|, u_3 = u_1 x u_2 (the set
//                                        of four poses MotionFromEssential forms does not depend on the signs an SVD picks).
// The reference's x86-64-v3 build contracts AngularError into FMAs (E x1, the squared norm, the dot product): they are
// written out with std::fma, as openmvg_b200/csrc/geom.cu writes them with __fma_rn.
#include "acransac_oracle.cpp"

namespace {

template <int N>
void jacobi_sym(double (*A)[N], double (*V)[N]) {
  for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0, diag = 0;
    for (int i = 0; i < N; ++i) { diag += A[i][i] * A[i][i]; for (int j = i + 1; j < N; ++j) off += A[i][j] * A[i][j]; }
    if (off <= 1e-60 * diag || off == 0.0) break;
    for (int p = 0; p < N - 1; ++p)
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
        for (int k = 0; k < N; ++k) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk; }
        for (int k = 0; k < N; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq; }
      }
  }
}

// b1, b2: all bearings [.][3]; s: ms sample indices; E row-major out
void angular_solve(bool upright, const double *b1, const double *b2, const uint32_t *s, double E[9]) {
  if (upright) {
    double A[4][4], V[4][4];
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) {
      double acc = 0;
      for (int t = 0; t < 3; ++t) {
        const double *a = b1 + 3 * (size_t)s[t], *b = b2 + 3 * (size_t)s[t];
        const double r[4] = {a[0] * b[1], -a[2] * b[1], -b[0] * a[1], -b[2] * a[1]};
        acc += r[i] * r[j];
      }
      A[i][j] = acc;
    }
    jacobi_sym<4>(A, V);
    int k = 0; for (int i = 1; i < 4; ++i) if (A[i][i] < A[k][k]) k = i;
    for (int i = 0; i < 9; ++i) E[i] = 0.0;
    E[1] = V[2][k]; E[3] = -V[0][k]; E[5] = V[1][k]; E[7] = V[3][k];
  } else {
    double A[9][9], f2[9];
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) {
      double acc = 0;
      for (int t = 0; t < 8; ++t) {
        const size_t q = s[t];
        acc += (b2[3 * q + i / 3] * b1[3 * q + i % 3]) * (b2[3 * q + j / 3] * b1[3 * q + j % 3]);
      }
      A[i][j] = acc;
    }
    smallest_two_eigvecs(A, E, f2);
  }
}

double angular_error(const double *E, const double *a, const double *b) {
  double m0 = std::fma(E[2], a[2], std::fma(E[1], a[1], E[0] * a[0]));
  double m1 = std::fma(E[5], a[2], std::fma(E[4], a[1], E[3] * a[0]));
  double m2 = std::fma(E[6], a[0], std::fma(E[8], a[2], E[7] * a[1]));
  const double z = std::fma(m2, m2, m0 * m0 + m1 * m1);
  if (z > 0.0) { const double sz = std::sqrt(z); m0 /= sz; m1 /= sz; m2 /= sz; }
  return std::fabs(std::asin(std::fma(m2, b[2], b[0] * m0 + b[1] * m1)));
}

double det3(const double (*m)[3]) {
  return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}

void motion_from_essential(const double *E, double R[4][9], double t[4][3]) {
  double M[3][3], V[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double v = 0; for (int k = 0; k < 3; ++k) v += E[3 * k + i] * E[3 * k + j]; M[i][j] = v; }
  jacobi_sym<3>(M, V);
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a) for (int b = 0; b < 2 - a; ++b) if (M[o[b + 1]][o[b + 1]] > M[o[b]][o[b]]) std::swap(o[b], o[b + 1]);
  double U[3][3], Vt[3][3];
  for (int c = 0; c < 3; ++c) for (int k = 0; k < 3; ++k) Vt[c][k] = V[k][o[c]];
  for (int c = 0; c < 2; ++c) {
    double u[3], n2 = 0;
    for (int r = 0; r < 3; ++r) { u[r] = E[3 * r] * Vt[c][0] + E[3 * r + 1] * Vt[c][1] + E[3 * r + 2] * Vt[c][2]; n2 += u[r] * u[r]; }
    const double n = std::sqrt(n2);
    for (int r = 0; r < 3; ++r) U[r][c] = u[r] / n;
  }
  U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
  U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
  U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
  if (det3(U) < 0) for (int r = 0; r < 3; ++r) U[r][2] = -U[r][2];
  if (det3(Vt) < 0) for (int k = 0; k < 3; ++k) Vt[2][k] = -Vt[2][k];
  const double W[2][3][3] = {{{0, -1, 0}, {1, 0, 0}, {0, 0, 1}}, {{0, 1, 0}, {-1, 0, 0}, {0, 0, 1}}};
  double Rw[2][9];
  for (int w = 0; w < 2; ++w) {
    double T[3][3];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += U[r][k] * W[w][k][c]; T[r][c] = v; }
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += T[r][k] * Vt[k][c]; Rw[w][3 * r + c] = v; }
  }
  const int PR[4] = {0, 1, 0, 1}, PT[4] = {0, 1, 1, 0};
  for (int p = 0; p < 4; ++p) {
    const double *Rp = Rw[PR[p]];
    const double s = PT[p] ? -1.0 : 1.0;
    const double tp[3] = {s * U[0][2], s * U[1][2], s * U[2][2]};
    double C[3];
    for (int i = 0; i < 3; ++i) { double v = 0; for (int k = 0; k < 3; ++k) v += -Rp[3 * k + i] * tp[k]; C[i] = v; }
    for (int i = 0; i < 3; ++i) { double v = 0; for (int k = 0; k < 3; ++k) v += Rp[3 * i + k] * C[k]; t[p][i] = -v; }
    for (int i = 0; i < 9; ++i) R[p][i] = Rp[i];
  }
}

double norm_cross(const double *a, const double *b) {
  const double c0 = a[1] * b[2] - a[2] * b[1], c1 = a[2] * b[0] - a[0] * b[2], c2 = a[0] * b[1] - a[1] * b[0];
  return std::sqrt(c0 * c0 + c1 * c1 + c2 * c2);
}

bool idw_midpoint_cheirality(const double *R, const double *t, const double *x0, const double *x1) {
  double Rx0[3];
  for (int i = 0; i < 3; ++i) Rx0[i] = R[3 * i] * x0[0] + R[3 * i + 1] * x0[1] + R[3 * i + 2] * x0[2];
  const double p = norm_cross(Rx0, x1), q = norm_cross(Rx0, t), r = norm_cross(x1, t);
  const double l0 = r / p, l1 = q / p;
  double e[4] = {0, 0, 0, 0};
  for (int i = 0; i < 3; ++i) {
    const double a = l0 * Rx0[i], b = l1 * x1[i];
    const double v0 = t[i] + a - b, v1 = t[i] + a + b, v2 = t[i] - a - b, v3 = t[i] - a + b;
    e[0] += v0 * v0; e[1] += v1 * v1; e[2] += v2 * v2; e[3] += v3 * v3;
  }
  // The reference takes std::min (vminsd), which fmin differs from only when an operand is NaN.  All four sums come from
  // the same l0, l1, t, Rx0, x1: a NaN in e[1..3] means a NaN l0 or l1, which makes e[0] NaN too, and then both forms
  // compare false.  With e[0] finite the two minima are equal.
  return e[0] < std::fmin(std::fmin(e[1], e[2]), e[3]);
}

// RelativePoseFromEssential: counts[4]; on true `sel` holds the chosen pose's list
bool relative_pose(const double *E, const double *b1, const double *b2, const uint32_t *idx, size_t n, int counts[4], std::vector<uint32_t> &sel) {
  double R[4][9], t[4][3];
  motion_from_essential(E, R, t);
  std::vector<uint32_t> lists[4];
  for (int p = 0; p < 4; ++p) {
    counts[p] = 0;
    for (size_t k = 0; k < n; ++k)
      if (idw_midpoint_cheirality(R[p], t[p], b1 + 3 * (size_t)idx[k], b2 + 3 * (size_t)idx[k])) { ++counts[p]; lists[p].push_back(idx[k]); }
  }
  sel.clear();
  const int best = (int)(std::max_element(counts, counts + 4) - counts);
  if (counts[best] == 0) return false;
  int sorted[4] = {counts[0], counts[1], counts[2], counts[3]};
  std::sort(sorted, sorted + 4);
  const double ratio = sorted[2] / static_cast<double>(sorted[3]);
  if (!(ratio < 0.7)) return false;
  sel = lists[best];
  return true;
}

}  // namespace

extern "C" {

// model 3: eight-point, 4: upright.  b1, b2 [n][ms][3]; E [n][9]
void oracle_angular_solver(int model, int n, const double *b1, const double *b2, double *E) {
  const bool upright = model == 4;
  const int ms = upright ? 3 : 8;
  const uint32_t s[8] = {0, 1, 2, 3, 4, 5, 6, 7};
  for (int k = 0; k < n; ++k) angular_solve(upright, b1 + 3 * ms * (size_t)k, b2 + 3 * ms * (size_t)k, s, E + 9 * (size_t)k);
}

// AngularError of candidate k: E [n][9], b1, b2 [n][3]
void oracle_angular_error(int n, const double *E, const double *b1, const double *b2, double *err) {
  for (int k = 0; k < n; ++k) err[k] = angular_error(E + 9 * (size_t)k, b1 + 3 * (size_t)k, b2 + 3 * (size_t)k);
}

void oracle_asin(int n, const double *x, double *y) {
  for (int k = 0; k < n; ++k) y[k] = std::asin(x[k]);
}

// four poses of MotionFromEssential: R [4][9] row-major, t [4][3] = translation()
void oracle_motion_from_essential(const double *E, double *R, double *t) {
  double r[4][9], tt[4][3];
  motion_from_essential(E, r, tt);
  std::memcpy(R, r, sizeof r); std::memcpy(t, tt, sizeof tt);
}

int oracle_relative_pose(const double *E, const double *b1, const double *b2, int n_index, const uint32_t *index,
                         int32_t *counts, uint32_t *selected, int32_t *n_selected) {
  int c[4]; std::vector<uint32_t> sel;
  const bool ok = relative_pose(E, b1, b2, index, (size_t)n_index, c, sel);
  for (int p = 0; p < 4; ++p) counts[p] = c[p];
  for (size_t k = 0; k < sel.size(); ++k) selected[k] = sel[k];
  *n_selected = (int32_t)sel.size();
  return ok;
}

// One pair of the filter.  ransac_inliers[n] / return value: the AC-RANSAC inliers; final_inliers[*n_final]: after
// RelativePoseFromEssential.  E [9], stats = {errorMax (radians), minNFA}, counts[4] the cheirality counts.
// trace (optional): {iterations run, models evaluated, iteration AC-RANSAC mode was entered or -1}.
int oracle_angular_acransac(int model, const double *b1, const double *b2, int n, double precision_deg, unsigned int iterations,
                            uint32_t *ransac_inliers, uint32_t *final_inliers, int32_t *n_final, double *E_out, double *stats,
                            int32_t *counts, int32_t *trace) {
  const bool upright = model == 4;
  double best_model[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  stats[0] = 0.0; stats[1] = 0.0; *n_final = 0;
  for (int p = 0; p < 4; ++p) counts[p] = 0;
  if (trace) { trace[0] = trace[1] = 0; trace[2] = -1; }
  std::vector<uint32_t> vec_inliers;
  Kernel K;
  K.n = n; K.model = -1; K.min_samples = upright ? 3 : 8; K.max_models = 1;
  K.logalpha0 = std::log10(1. / 2.); K.mult_error = 1. / 4.;
  const unsigned int sizeSample = (unsigned int)K.min_samples, nData = (unsigned int)n;
  if (nData > sizeSample) {
    const double inf = std::numeric_limits<double>::infinity();
    const double maxThreshold = precision_deg * M_PI / 180.0;          // ACRANSAC(kernel, ..., D2R(precision)), N2 = I
    std::vector<uint32_t> vec_index(nData); for (unsigned int i = 0; i < nData; ++i) vec_index[i] = i;
    std::vector<uint32_t> vec_sample(sizeSample);
    NFA nfa(K, maxThreshold, true);
    double minNFA = inf, errorMax = inf;
    int nIterReserve = (int)(iterations / 10);
    unsigned int nIter = iterations - nIterReserve;
    bool bACRansacMode = false;
    MT19937 rng(5489u);
    unsigned int iter = 0;
    for (iter = 0; iter < nIter && iter < iterations; ++iter) {
      if (bACRansacMode) uniform_sample_shuffle(sizeSample, rng, vec_index, vec_sample);
      else uniform_sample_reject(sizeSample, nData, rng, vec_sample);
      double Em[9];
      angular_solve(upright, b1, b2, vec_sample.data(), Em);
      bool better = false;
      for (unsigned int i = 0; i < nData; ++i) { const double a = angular_error(Em, b1 + 3 * (size_t)i, b2 + 3 * (size_t)i); nfa.residuals[i] = a * a; }
      if (!bACRansacMode) {
        unsigned int nInlier = 0;
        for (unsigned int i = 0; i < nData; ++i) if (nfa.residuals[i] <= maxThreshold) ++nInlier;
        if (nInlier > 2.5 * sizeSample) { bACRansacMode = true; if (trace) trace[2] = (int)iter; }
      }
      if (bACRansacMode) {
        std::pair<double, double> nfa_threshold(minNFA, 0.0);
        if (nfa.compute(vec_inliers, nfa_threshold)) {
          better = true; minNFA = nfa_threshold.first; errorMax = nfa_threshold.second;
          std::memcpy(best_model, Em, sizeof best_model);
        }
      }
      if (!bACRansacMode && (int)iter > nIterReserve * 2) { nIter = 0; continue; }
      if (bACRansacMode && ((better && minNFA < 0) || ((iter + 1) == nIter && nIterReserve > 0))) {
        if (vec_inliers.empty()) { ++nIter; --nIterReserve; }
        else {
          vec_index = vec_inliers;
          if (nIterReserve) { nIter = iter + 1 + nIterReserve; nIterReserve = 0; }
        }
      }
    }
    if (trace) { trace[0] = (int)iter; trace[1] = (int)iter; }
    if (minNFA >= 0) vec_inliers.clear();
    if (!vec_inliers.empty()) errorMax = std::sqrt(errorMax);             // unormalizeError
    stats[0] = errorMax; stats[1] = minNFA;
  }
  for (size_t i = 0; i < vec_inliers.size(); ++i) ransac_inliers[i] = vec_inliers[i];
  std::vector<uint32_t> sel;
  int c[4];
  relative_pose(best_model, b1, b2, vec_inliers.data(), vec_inliers.size(), c, sel);
  for (int p = 0; p < 4; ++p) counts[p] = c[p];
  for (size_t i = 0; i < sel.size(); ++i) final_inliers[i] = sel[i];
  *n_final = (int32_t)sel.size();
  for (int i = 0; i < 9; ++i) E_out[i] = best_model[i];
  return (int)vec_inliers.size();
}

}  // extern "C"
