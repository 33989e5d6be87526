// essential_oracle.cpp — CPU restatement of the essential-matrix geometric filter (five-point AC-RANSAC) that
// openMVG_main_GeometricFilter runs with `-g e` (SURVEY §8f N4, DESIGN §3.8).
//
// TEST INFRASTRUCTURE ONLY.  Built as its own library (oracle/_build/liboracle_essential.so, oracle/essential.mk); it
// includes acransac_oracle.cpp for the parts the F/H filter already restates: MT19937 + Lemire, the two UniformSample
// variants, the NFA tables and the quantified NFA.
//
// Parity status: PINNED by tests/test_oracle_geom_essential.py against oracle/_ref/libref_geom_essential.so (the
// reference's own FivePointsRelativePose and ACRANSAC + ACKernelAdaptorEssential<FivePointSolver,
// EpipolarDistanceError>): the same SET of solutions per five-point sample (up to scale and sign), identical inlier
// lists, (errorMax, minNFA) to 1e-9, E equal up to scale to 1e-7.
//
// Reference lines restated ($OPENMVG/src/openMVG):
//   matching_image_collection/E_ACRobust.hpp:55-150                    Robust_estimation (skips, kernel, keep rule)
//   robust_estimation/robust_estimator_ACRansacKernelAdaptator.hpp:294-380   ACKernelAdaptorEssential
//   multiview/solver_essential_five_point.cpp:35-214                   FivePointsRelativePose
//   multiview/essential.cpp:48-53                                      FundamentalFromEssential
//   cameras/Camera_Pinhole.hpp:136-139                                 bearing = normalize(K^-1 [x; 1])
// The linear algebra the reference takes from Eigen is restated from the published algorithms instead:
//   SelfAdjointEigenSolver<9x9> -> cyclic Jacobi (any orthonormal basis of the 4-D null space spans the same E family);
//   FullPivLU solve             -> Gauss-Jordan elimination with partial pivoting;
//   EigenSolver<10x10>          -> Householder reduction to Hessenberg form + Francis double-shift QR with the
//                                  EISPACK exceptional shifts (Golub & Van Loan §7.5); a 2x2 diagonal block is a
//                                  complex pair iff its discriminant is negative, as in the reference; the
//                                  eigenvector of a real eigenvalue is the null vector of At - lambda I
//                                  (Gaussian elimination with complete pivoting, last unknown = 1).
// openmvg_b200/csrc/geom.cu runs the same arithmetic, entry by entry, with the row/column loops spread over a warp.
#include "acransac_oracle.cpp"

namespace {

// eigenvectors of the 4 smallest eigenvalues of a symmetric 9x9 (same cyclic Jacobi as the F path), as basis[9][4]
void smallest_four_eigvecs(double A[9][9], double basis[9][4]) {
  double V[9][9];
  for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0, diag = 0;
    for (int i = 0; i < 9; ++i) { diag += A[i][i] * A[i][i]; for (int j = i + 1; j < 9; ++j) off += A[i][j] * A[i][j]; }
    if (off <= 1e-60 * diag || off == 0.0) break;
    for (int p = 0; p < 8; ++p)
      for (int q = p + 1; q < 9; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 9; ++k) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
        for (int k = 0; k < 9; ++k) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk; }
        for (int k = 0; k < 9; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq; }
      }
  }
  unsigned used = 0;
  for (int c = 0; c < 4; ++c) {
    int best = -1;
    for (int i = 0; i < 9; ++i) if (!(used >> i & 1u) && (best < 0 || A[i][i] < A[best][best])) best = i;
    used |= 1u << best;
    for (int k = 0; k < 9; ++k) basis[k][c] = V[k][best];
  }
}

// Polynomials in (x, y, z) in the monomial order of Stewenius et al.: cubic terms 0-9 (xxx xxy xyy yyy xxz xyz yyz
// xzz yzz zzz), quadratic 10-15 (xx xy yy xz yz zz), linear 16-18 (x y z), constant 19.  A linear polynomial is
// held as its 4 trailing coefficients (x y z 1), a quadratic as its 10 trailing ones (xx .. 1).
void poly_lin_lin(const double a[4], const double b[4], double r[10]) {
  r[0] = a[0] * b[0];
  r[1] = a[0] * b[1] + a[1] * b[0];
  r[2] = a[1] * b[1];
  r[3] = a[0] * b[2] + a[2] * b[0];
  r[4] = a[1] * b[2] + a[2] * b[1];
  r[5] = a[2] * b[2];
  r[6] = a[0] * b[3] + a[3] * b[0];
  r[7] = a[1] * b[3] + a[3] * b[1];
  r[8] = a[2] * b[3] + a[3] * b[2];
  r[9] = a[3] * b[3];
}
void poly_quad_lin(const double a[10], const double b[4], double r[20]) {
  const double xx = a[0], xy = a[1], yy = a[2], xz = a[3], yz = a[4], zz = a[5], x = a[6], y = a[7], z = a[8], o = a[9];
  const double bx = b[0], by = b[1], bz = b[2], bo = b[3];
  r[0] = xx * bx;
  r[1] = xx * by + xy * bx;
  r[2] = xy * by + yy * bx;
  r[3] = yy * by;
  r[4] = xx * bz + xz * bx;
  r[5] = xy * bz + yz * bx + xz * by;
  r[6] = yy * bz + yz * by;
  r[7] = xz * bz + zz * bx;
  r[8] = yz * bz + zz * by;
  r[9] = zz * bz;
  r[10] = xx * bo + x * bx;
  r[11] = xy * bo + x * by + y * bx;
  r[12] = yy * bo + y * by;
  r[13] = xz * bo + x * bz + z * bx;
  r[14] = yz * bo + y * bz + z * by;
  r[15] = zz * bo + z * bz;
  r[16] = x * bo + o * bx;
  r[17] = y * bo + o * by;
  r[18] = z * bo + o * bz;
  r[19] = o * bo;
}

// E(x,y,z) = x B0 + y B1 + z B2 + B3 (B = basis columns, E_ij = row 3i+j).  Row 0: det E = 0 (Nister eq. 19);
// rows 1 + 3i + j: (E E^T - tr(E E^T)/2 I) E = 0 (eqs. 20-23).
void eet_entry(const double E[9][4], int i, int j, double r[10]) {
  double t[10];
  poly_lin_lin(E[3 * i], E[3 * j], r);
  for (int k = 1; k < 3; ++k) { poly_lin_lin(E[3 * i + k], E[3 * j + k], t); for (int c = 0; c < 10; ++c) r[c] += t[c]; }
}
void det_row(const double E[9][4], double row[20]) {
  static const int T[3][4] = {{1, 5, 2, 4}, {2, 3, 0, 5}, {0, 4, 1, 3}};   // cofactor of column c: E0a E1b - E0d E1e
  for (int c = 0; c < 20; ++c) row[c] = 0;
  for (int c = 0; c < 3; ++c) {
    double u[10], v[10], w[20];
    poly_lin_lin(E[T[c][0]], E[T[c][1]], u); poly_lin_lin(E[T[c][2]], E[T[c][3]], v);
    for (int k = 0; k < 10; ++k) u[k] -= v[k];
    poly_quad_lin(u, E[6 + c], w);
    for (int k = 0; k < 20; ++k) row[k] += w[k];
  }
}
void trace_row(const double L[6][10], const double E[9][4], int i, int j, double row[20]) {
  static const int S[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};            // symmetric L[i][k] -> packed upper index
  double w[20];
  poly_quad_lin(L[S[i][0]], E[j], row);
  for (int k = 1; k < 3; ++k) { poly_quad_lin(L[S[i][k]], E[3 * k + j], w); for (int c = 0; c < 20; ++c) row[c] += w[c]; }
}
void constraint_matrix(const double E[9][4], double C[10][20]) {
  static const int P[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
  double L[6][10];
  for (int t = 0; t < 6; ++t) eet_entry(E, P[t][0], P[t][1], L[t]);
  for (int c = 0; c < 10; ++c) {
    const double half_trace = 0.5 * (L[0][c] + L[3][c] + L[5][c]);
    L[0][c] -= half_trace; L[3][c] -= half_trace; L[5][c] -= half_trace;
  }
  det_row(E, C[0]);
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) trace_row(L, E, i, j, C[1 + 3 * i + j]);
}

// [C1 | C2] -> C1^-1 C2 by Gauss-Jordan elimination with partial pivoting (first maximum wins)
void gauss_jordan(double C[10][20], double M[10][10]) {
  for (int k = 0; k < 10; ++k) {
    int piv = k;
    for (int r = k + 1; r < 10; ++r) if (std::fabs(C[r][k]) > std::fabs(C[piv][k])) piv = r;
    if (piv != k) for (int j = 0; j < 20; ++j) std::swap(C[k][j], C[piv][j]);
    double f[10];
    for (int r = 0; r < 10; ++r) f[r] = r == k ? 0.0 : C[r][k] / C[k][k];
    for (int j = k; j < 20; ++j) for (int r = 0; r < 10; ++r) if (r != k) C[r][j] -= f[r] * C[k][j];
  }
  for (int r = 0; r < 10; ++r) for (int j = 0; j < 10; ++j) M[r][j] = C[r][10 + j] / C[r][r];
}

// Householder reduction of a 10x10 to upper Hessenberg form (similarity; the reflectors are not kept)
void hessenberg(double a[10][10]) {
  const int n = 10;
  for (int m = 1; m < n - 1; ++m) {
    double scale = 0;
    for (int i = m; i < n; ++i) scale += std::fabs(a[i][m - 1]);
    if (scale == 0.0) continue;
    double u[10], h = 0;
    for (int i = n - 1; i >= m; --i) { u[i] = a[i][m - 1] / scale; h += u[i] * u[i]; }
    const double g = u[m] > 0 ? -std::sqrt(h) : std::sqrt(h);
    h -= u[m] * g; u[m] -= g;
    for (int j = m; j < n; ++j) {                      // (I - u u'/h) A
      double f = 0;
      for (int i = n - 1; i >= m; --i) f += u[i] * a[i][j];
      f /= h;
      for (int i = m; i < n; ++i) a[i][j] -= f * u[i];
    }
    for (int i = 0; i < n; ++i) {                      // A (I - u u'/h)
      double f = 0;
      for (int j = n - 1; j >= m; --j) f += u[j] * a[i][j];
      f /= h;
      for (int j = m; j < n; ++j) a[i][j] -= f * u[j];
    }
    a[m][m - 1] = scale * g;
    for (int i = m + 1; i < n; ++i) a[i][m - 1] = 0.0;
  }
}

// Francis double-shift QR on an upper Hessenberg 10x10 (eigenvalues only), with EISPACK's budget of 30 n iterations
// for the whole matrix.  false: no convergence (the sample then yields no model).
bool hessenberg_qr(double a[10][10], double wr[10], double wi[10]) {
  const int n = 10;
  double anorm = 0;
  for (int i = 0; i < n; ++i) for (int j = std::max(i - 1, 0); j < n; ++j) anorm += std::fabs(a[i][j]);
  int nn = n - 1, itn = 30 * n;
  double t = 0;
  while (nn >= 0) {
    int its = 0, l;
    do {
      for (l = nn; l >= 1; --l) {                      // a negligible subdiagonal entry splits the matrix
        double s = std::fabs(a[l - 1][l - 1]) + std::fabs(a[l][l]);
        if (s == 0.0) s = anorm;
        if (std::fabs(a[l][l - 1]) + s == s) { a[l][l - 1] = 0.0; break; }
      }
      double x = a[nn][nn];
      if (l == nn) { wr[nn] = x + t; wi[nn] = 0.0; --nn; continue; }
      double y = a[nn - 1][nn - 1], w = a[nn][nn - 1] * a[nn - 1][nn];
      if (l == nn - 1) {                               // a 2x2 block: real pair iff the discriminant is >= 0
        const double p = 0.5 * (y - x), q = p * p + w;
        double z = std::sqrt(std::fabs(q));
        x += t;
        if (q >= 0.0) {
          z = p + (p >= 0 ? z : -z);
          wr[nn - 1] = wr[nn] = x + z;
          if (z != 0.0) wr[nn] = x - w / z;
          wi[nn - 1] = wi[nn] = 0.0;
        } else {
          wr[nn - 1] = wr[nn] = x + p;
          wi[nn - 1] = -z; wi[nn] = z;
        }
        nn -= 2;
        continue;
      }
      if (itn == 0) return false;
      if (its == 10 || its == 20) {                    // exceptional shift
        t += x;
        for (int i = 0; i <= nn; ++i) a[i][i] -= x;
        const double s = std::fabs(a[nn][nn - 1]) + std::fabs(a[nn - 1][nn - 2]);
        y = x = 0.75 * s;
        w = -0.4375 * s * s;
      }
      ++its; --itn;
      int m;
      double p = 0, q = 0, r = 0, z;
      for (m = nn - 2; m >= l; --m) {                  // two consecutive small subdiagonal entries
        z = a[m][m];
        r = x - z;
        double s = y - z;
        p = (r * s - w) / a[m + 1][m] + a[m][m + 1];
        q = a[m + 1][m + 1] - z - r - s;
        r = a[m + 2][m + 1];
        s = std::fabs(p) + std::fabs(q) + std::fabs(r);
        p /= s; q /= s; r /= s;
        if (m == l) break;
        const double u = std::fabs(a[m][m - 1]) * (std::fabs(q) + std::fabs(r));
        const double v = std::fabs(p) * (std::fabs(a[m - 1][m - 1]) + std::fabs(z) + std::fabs(a[m + 1][m + 1]));
        if (u + v == v) break;
      }
      for (int i = m + 2; i <= nn; ++i) { a[i][i - 2] = 0.0; if (i != m + 2) a[i][i - 3] = 0.0; }
      for (int k = m; k <= nn - 1; ++k) {              // chase the bulge
        if (k != m) {
          p = a[k][k - 1]; q = a[k + 1][k - 1]; r = 0.0;
          if (k != nn - 1) r = a[k + 2][k - 1];
          x = std::fabs(p) + std::fabs(q) + std::fabs(r);
          if (x != 0.0) { p /= x; q /= x; r /= x; }
        }
        const double sq = std::sqrt(p * p + q * q + r * r), s = p >= 0 ? sq : -sq;
        if (s == 0.0) continue;
        if (k == m) { if (l != m) a[k][k - 1] = -a[k][k - 1]; }
        else a[k][k - 1] = -s * x;
        p += s; x = p / s; y = q / s; z = r / s; q /= p; r /= p;
        for (int j = k; j <= nn; ++j) {                // rows k..k+2
          double pp = a[k][j] + q * a[k + 1][j];
          if (k != nn - 1) { pp += r * a[k + 2][j]; a[k + 2][j] -= pp * z; }
          a[k + 1][j] -= pp * y; a[k][j] -= pp * x;
        }
        const int mmin = nn < k + 3 ? nn : k + 3;
        for (int i = l; i <= mmin; ++i) {              // columns k..k+2
          double pp = x * a[i][k] + y * a[i][k + 1];
          if (k != nn - 1) { pp += z * a[i][k + 2]; a[i][k + 2] -= pp * r; }
          a[i][k + 1] -= pp * q; a[i][k] -= pp;
        }
      }
    } while (l < nn - 1);
  }
  return true;
}

// null vector of (At - lambda I) by Gaussian elimination with complete pivoting; the last unknown is set to 1
void null_vector(const double At[10][10], double lambda, double v[10]) {
  double W[10][10]; int cp[10];
  for (int i = 0; i < 10; ++i) { cp[i] = i; for (int j = 0; j < 10; ++j) W[i][j] = At[i][j] - (i == j ? lambda : 0.0); }
  for (int k = 0; k < 9; ++k) {
    int pr = k, pc = k;
    for (int r = k; r < 10; ++r) for (int c = k; c < 10; ++c) if (std::fabs(W[r][c]) > std::fabs(W[pr][pc])) { pr = r; pc = c; }
    if (pr != k) for (int c = 0; c < 10; ++c) std::swap(W[k][c], W[pr][c]);
    if (pc != k) { for (int r = 0; r < 10; ++r) std::swap(W[r][k], W[r][pc]); std::swap(cp[k], cp[pc]); }
    for (int r = k + 1; r < 10; ++r) {
      const double f = W[r][k] / W[k][k];
      for (int c = k; c < 10; ++c) W[r][c] -= f * W[k][c];
    }
  }
  double y[10];
  y[9] = 1.0;
  for (int i = 8; i >= 0; --i) {
    double s = 0;
    for (int j = i + 1; j < 10; ++j) s += W[i][j] * y[j];
    y[i] = -s / W[i][i];
  }
  for (int i = 0; i < 10; ++i) v[cp[i]] = y[i];
}

// multiview/solver_essential_five_point.cpp:170-212.  b1, b2: 5 bearing pairs [5][3].  E: up to 10 models, row-major,
// each satisfying b2' E b1 = 0 (the reference's E.transpose() of its column-major map).
int five_point(const double b1[5][3], const double b2[5][3], double Es[10][9]) {
  double AtA[9][9];                                     // EncodeEpipolarEquation: row = [x2(0) x1', x2(1) x1', x2(2) x1']
  for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) {
    double acc = 0;
    for (int t = 0; t < 5; ++t) acc += (b2[t][i / 3] * b1[t][i % 3]) * (b2[t][j / 3] * b1[t][j % 3]);
    AtA[i][j] = acc;
  }
  double E[9][4];
  smallest_four_eigvecs(AtA, E);
  double C[10][20], M[10][10];
  constraint_matrix(E, C);
  gauss_jordan(C, M);
  double At[10][10] = {};                               // the action matrix of the reference
  static const int R[6] = {0, 1, 2, 4, 5, 7};
  for (int r = 0; r < 6; ++r) for (int c = 0; c < 10; ++c) At[r][c] = M[R[r]][c];
  At[6][0] = At[7][1] = At[8][3] = At[9][6] = -1.0;
  double H[10][10], wr[10], wi[10];
  std::memcpy(H, At, sizeof H);
  hessenberg(H);
  if (!hessenberg_qr(H, wr, wi)) return 0;
  int n = 0;
  for (int s = 0; s < 10; ++s) {
    if (wi[s] != 0.0) continue;
    double v[10];
    null_vector(At, wr[s], v);
    for (int k = 0; k < 9; ++k) Es[n][k] = E[k][0] * v[6] + E[k][1] * v[7] + E[k][2] * v[8] + E[k][3] * v[9];
    ++n;
  }
  return n;
}

// Pinhole_Intrinsic::operator(): normalize(K^-1 [x; y; 1]), K = [[f, 0, ppx], [0, f, ppy], [0, 0, 1]]
void bearing(double f, double ppx, double ppy, double x, double y, double b[3]) {
  const double u = (x - ppx) / f, v = (y - ppy) / f;
  const double nrm = std::sqrt(u * u + v * v + 1.0);
  b[0] = u / nrm; b[1] = v / nrm; b[2] = 1.0 / nrm;
}

// FundamentalFromEssential: F = K_J^-T E K_I^-1, K^-1 = [[1/f, 0, -ppx/f], [0, 1/f, -ppy/f], [0, 0, 1]]
void fundamental_from_essential(const double E[9], const double intr[6], double F[9]) {
  const double KI[9] = {1.0 / intr[0], 0, -intr[1] / intr[0], 0, 1.0 / intr[0], -intr[2] / intr[0], 0, 0, 1.0};
  const double KJ[9] = {1.0 / intr[3], 0, -intr[4] / intr[3], 0, 1.0 / intr[3], -intr[5] / intr[3], 0, 0, 1.0};
  double T[9];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += KJ[3 * k + r] * E[3 * k + c]; T[3 * r + c] = v; }
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += T[3 * r + k] * KI[3 * k + c]; F[3 * r + c] = v; }
}

}  // namespace

extern "C" {

// b1, b2: n samples of 5 bearing pairs [n][5][3]; E: [n][10][9]; n_models[n]
void oracle_five_point(int n, const double *b1, const double *b2, double *E, int32_t *n_models) {
  for (int s = 0; s < n; ++s) {
    double Es[10][9];
    const int k = five_point(reinterpret_cast<const double(*)[3]>(b1 + 15 * s), reinterpret_cast<const double(*)[3]>(b2 + 15 * s), Es);
    n_models[s] = k;
    for (int m = 0; m < k; ++m) for (int t = 0; t < 9; ++t) E[90 * s + 9 * m + t] = Es[m][t];
  }
}

// Same contract as ref_acransac_essential (oracle/ref_geom_essential_driver.cpp).  intr = {f, ppx, ppy} of I then J.
// stats = {errorMax (SQUARED pixels, as the reference leaves it), minNFA}.  trace (optional): {iterations run,
// models evaluated, iteration at which AC-RANSAC mode was entered or -1, samples without a model}.
int oracle_acransac_essential(const double *xI, const double *xJ, int n, int wI, int hI, int wJ, int hJ, const double *intr,
                              double precision, unsigned int iterations, uint32_t *inliers_out, double *E_out, double *stats, int *trace) {
  std::vector<uint32_t> vec_inliers;
  double best_model[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  stats[0] = 0.0; stats[1] = 0.0;
  for (int i = 0; i < 9; ++i) E_out[i] = best_model[i];
  if (trace) { trace[0] = trace[1] = trace[3] = 0; trace[2] = -1; }
  const unsigned int sizeSample = 5, nData = (unsigned int)n;
  if (nData <= sizeSample) return 0;
  Kernel K;                                              // only what NFA reads: no normalisation (N1 = N2 = I)
  K.n = n; K.model = 2; K.min_samples = 5; K.max_models = 10; K.mult_error = 0.5;
  K.logalpha0 = std::log10(2. * std::hypot((double)wJ, (double)hJ) / (wJ * (double)hJ) / 0.5);
  std::vector<double> b1(3 * n), b2(3 * n);
  for (int i = 0; i < n; ++i) {
    bearing(intr[0], intr[1], intr[2], xI[2 * i], xI[2 * i + 1], &b1[3 * i]);
    bearing(intr[3], intr[4], intr[5], xJ[2 * i], xJ[2 * i + 1], &b2[3 * i]);
  }
  const double inf = std::numeric_limits<double>::infinity();
  const double maxThreshold = precision * precision;
  std::vector<uint32_t> vec_index(nData); for (unsigned int i = 0; i < nData; ++i) vec_index[i] = i;
  std::vector<uint32_t> vec_sample(sizeSample);
  NFA nfa(K, maxThreshold, true);
  double minNFA = inf, errorMax = inf;
  int nIterReserve = (int)(iterations / 10);
  unsigned int nIter = iterations - nIterReserve;
  bool bACRansacMode = false;
  MT19937 rng(5489u);
  unsigned int iter = 0; int n_models = 0, n_empty = 0;
  for (iter = 0; iter < nIter && iter < iterations; ++iter) {
    if (bACRansacMode) uniform_sample_shuffle(sizeSample, rng, vec_index, vec_sample);
    else uniform_sample_reject(sizeSample, nData, rng, vec_sample);
    double s1[5][3], s2[5][3], Es[10][9];
    for (int t = 0; t < 5; ++t) for (int c = 0; c < 3; ++c) { s1[t][c] = b1[3 * vec_sample[t] + c]; s2[t][c] = b2[3 * vec_sample[t] + c]; }
    const int nm = five_point(s1, s2, Es);
    n_empty += nm == 0;
    bool better = false;
    for (int mi = 0; mi < nm; ++mi) {
      ++n_models;
      double F[9];
      fundamental_from_essential(Es[mi], intr, F);
      for (unsigned int i = 0; i < nData; ++i) nfa.residuals[i] = epipolar_error(F, xI[2 * i], xI[2 * i + 1], xJ[2 * i], xJ[2 * i + 1]);
      if (!bACRansacMode) {
        unsigned int nInlier = 0;
        for (unsigned int i = 0; i < nData; ++i) if (nfa.residuals[i] <= maxThreshold) ++nInlier;
        if (nInlier > 2.5 * sizeSample) { bACRansacMode = true; if (trace) trace[2] = (int)iter; }
      }
      if (bACRansacMode) {
        std::pair<double, double> nfa_threshold(minNFA, 0.0);
        if (nfa.compute(vec_inliers, nfa_threshold)) {
          better = true; minNFA = nfa_threshold.first; errorMax = nfa_threshold.second;
          std::memcpy(best_model, Es[mi], sizeof best_model);
        }
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
  if (trace) { trace[0] = (int)iter; trace[1] = n_models; trace[3] = n_empty; }
  if (minNFA >= 0) vec_inliers.clear();
  for (size_t i = 0; i < vec_inliers.size(); ++i) inliers_out[i] = vec_inliers[i];
  for (int i = 0; i < 9; ++i) E_out[i] = best_model[i];
  stats[0] = errorMax; stats[1] = minNFA;             // unormalizeError is the identity: errorMax stays squared
  return (int)vec_inliers.size();
}

}  // extern "C"
