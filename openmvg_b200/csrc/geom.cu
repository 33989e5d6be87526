// geom.cu — per-pair a-contrario RANSAC (fundamental-matrix, homography, essential-matrix and angular essential-matrix models) on sm_90a: the
// geometric filter openMVG runs right after putative matching (SURVEY §8f N4).
//
// Replaces (reference, $OPENMVG/src/openMVG):
//   matching_image_collection/GeometricFilter.hpp:66-128          the pair loop (OpenMP over pairs)
//   matching_image_collection/F_ACRobust.hpp:45-106               GeometricFilter_FMatrix_AC::Robust_estimation
//   robust_estimation/robust_estimator_ACRansac.hpp:57-119,190-300,303-490   logcombi, NFA, ACRANSAC
//   robust_estimation/rand_sampling.hpp:35-95                     the two UniformSample variants
//   robust_estimation/robust_estimator_ACRansacKernelAdaptator.hpp:43-63,120-200
//   multiview/conditioning.cpp:54-77, solver_fundamental_kernel.cpp:38-95,157-166, numeric/poly.h:32-96
//
// AC-RANSAC is sequential per pair (the sampling set of iteration k is the inlier set of the best model so far, the
// std::mt19937 stream is consumed in order), so the parallelism is ACROSS pairs — one CTA per pair, thousands of
// pairs per launch — and, inside a pair, across the matches (residuals, the 20-bin NFA histogram, the ordered
// inlier compaction).  The control flow, the generator (MT19937 + libstdc++'s Lemire down-scaling) and every
// floating-point expression that feeds a comparison follow the CPU restatement used by the tests (acransac_oracle.cpp) line by line; this file is
// compiled with -fmad=false so those expressions round exactly as the CPU evaluates them.
#include "common.cuh"

#include <cfloat>
#include <cmath>
#include <type_traits>
#include <vector>

namespace omvg { namespace geom {

constexpr int THREADS = 128;
constexpr int NBINS = 20;

struct Rng { uint32_t *mt; int idx; };        // state in shared memory, driven by thread 0
__device__ void rng_seed(Rng &g, uint32_t seed) { g.mt[0] = seed; for (int i = 1; i < 624; ++i) g.mt[i] = 1812433253u * (g.mt[i - 1] ^ (g.mt[i - 1] >> 30)) + (uint32_t)i; g.idx = 624; }
__device__ uint32_t rng_next(Rng &g) {
  if (g.idx >= 624) {
    for (int i = 0; i < 624; ++i) {
      const uint32_t y = (g.mt[i] & 0x80000000u) | (g.mt[(i + 1) % 624] & 0x7fffffffu);
      g.mt[i] = g.mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    g.idx = 0;
  }
  uint32_t y = g.mt[g.idx++];
  y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
  return y;
}
// std::uniform_int_distribution<uint32_t> of libstdc++ 13 on a 32-bit generator (Lemire), value - a
__device__ uint32_t lemire(Rng &g, uint32_t range) {
  unsigned long long product = (unsigned long long)rng_next(g) * (unsigned long long)range;
  uint32_t low = (uint32_t)product;
  if (low < range) {
    const uint32_t threshold = (0u - range) % range;
    while (low < threshold) { product = (unsigned long long)rng_next(g) * (unsigned long long)range; low = (uint32_t)product; }
  }
  return (uint32_t)(product >> 32);
}

// numeric/poly.h:32-96
__device__ int solve_cubic(double a, double b, double c, double x[3]) {
  const double eps = DBL_EPSILON;
  a /= 3;
  double p = (b - 3 * a * a) / 3;
  double q = (2 * a * a * a - a * b + c) / 2;
  double d = q * q + p * p * p;
  const double tolq = fmax(fabs(2 * a * a * a), fmax(fabs(a * b), fabs(c)));
  const double tolp = fmax(fabs(b), fabs(3 * a * a));
  int n = (d > eps * fmax(p * p * tolp, fabs(q) * tolq) ? 1 : 3);
  if (n == 1) {
    d = pow(fabs(q) + sqrt(d), 1 / (double)3);
    x[0] = d - p / d;
    if (q > 0) x[0] = -x[0];
  } else {
    if (3 * p >= -eps * tolp) { n = 1; x[0] = 0; }
    else {
      p = sqrt(-p);
      q /= p * p * p;
      d = (q <= -1) ? 3.14159265358979323846 : (q >= 1) ? 0 : acos(q);
      for (int i = 0; i < 3; ++i) x[i] = -2 * p * cos((d + 2 * 3.14159265358979323846 * i) / 3);
    }
  }
  for (int i = 0; i < n; ++i) x[i] -= a;
  return n;
}

// cyclic Jacobi on a symmetric 9x9 in shared memory (thread 0), eigenvectors of the two smallest eigenvalues
__device__ void smallest_two_eigvecs(double (*A)[9], double (*V)[9], double f1[9], double f2[9]) {
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
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 9; ++k) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
        for (int k = 0; k < 9; ++k) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk; }
        for (int k = 0; k < 9; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq; }
      }
  }
  int i1 = 0; for (int i = 1; i < 9; ++i) if (A[i][i] < A[i1][i1]) i1 = i;
  int i2 = i1 == 0 ? 1 : 0; for (int i = 0; i < 9; ++i) if (i != i1 && A[i][i] < A[i2][i2]) i2 = i;
  for (int k = 0; k < 9; ++k) { f1[k] = V[k][i1]; f2[k] = V[k][i2]; }
}

__device__ __forceinline__ double epipolar_error(const double *F, double x, double y, double u, double v) {
  const double fx0 = F[0] * x + F[1] * y + F[2], fx1 = F[3] * x + F[4] * y + F[5], fx2 = F[6] * x + F[7] * y + F[8];
  const double dt = fx0 * u + fx1 * v + fx2;
  return dt * dt / (fx0 * fx0 + fx1 * fx1);
}

// solver_homography_kernel.hpp:59-63
__device__ __forceinline__ double transfer_error(const double *H, double x, double y, double u, double v) {
  const double p0 = H[0] * x + H[1] * y + H[2], p1 = H[3] * x + H[4] * y + H[5], p2 = H[6] * x + H[7] * y + H[8];
  const double dx = u - p0 / p2, dy = v - p1 / p2;
  return dx * dx + dy * dy;
}
__device__ __forceinline__ double model_error(int model, const double *M, double x, double y, double u, double v) {
  return model == 0 ? epipolar_error(M, x, y, u, v) : transfer_error(M, x, y, u, v);
}

struct Args {
  const unsigned long long *offsets;       // [n_pairs + 1] into the match arrays
  const double *xI, *xJ;                   // [n_matches][2] pixels
  const int *image_size;                   // [n_pairs][4] wI hI wJ hJ
  double precision; unsigned int iterations; int model;   // model 0: fundamental (7 points, <= 3 models), 1: homography (4 points, 1 model)
  double *x1, *x2;                         // scratch [n_matches][2]: normalised points
  float *logc_n, *logc_k, *l10;            // scratch [n_matches + n_pairs] each (n + 1 entries per pair)
  uint32_t *vec_index;                     // scratch [n_matches]
  uint32_t *inliers;                       // out [n_matches]: first n_inliers[p] entries of pair p's segment
  uint32_t *n_inliers; double *F; double *stats;
  unsigned int n_pairs;
  const double *intr;                      // essential model: [n_pairs][6] f, ppx, ppy of view I then view J
};

struct Smem {
  uint32_t mt[624];
  double AtA[9][9], V[9][9], f1[9], f2[9], models[3][9];
  double N1[9], N2[9];
  int hist[NBINS]; int n_le; int warp_cnt[THREADS / 32];
  uint32_t sample[7];
  int n_models, better_now;
  double nfa_thr, nfa_val;                 // threshold / NFA of the model being accepted
};

// ---------------------------------------------------------------- essential model: the five-point solver (DESIGN §3.8)
// multiview/solver_essential_five_point.cpp:35-214, restated step by step as the CPU restatement used by the tests (essential_oracle.cpp) does it (same
// algorithms, same operation order per entry).  One warp solves one sample; every row- or column-parallel loop is spread
// over the lanes, the scalar control flow runs redundantly in all lanes, and shared scalars are written by lane 0.
struct FivePointWork {
  double AtA[9][9], V[9][9], basis[9][4];  // A'A of the 5 epipolar rows, Jacobi vectors, the 4-D null space (E_ij = row 3i+j)
  double L[6][10], C[10][20], f[10];       // E E' - tr/2 (packed upper), the 10x20 constraint matrix, elimination factors
  double At[10][10], H[10][10];            // the action matrix and its Hessenberg / quasi-triangular form
  double models[10][9];                    // real solutions, row-major (b2' E b1 = 0)
  int n_models;
};

// Polynomials in (x, y, z), monomials in the order of Stewenius et al. (cubic 0-9, quadratic 10-15, x y z 16-18, 1 19);
// a linear polynomial is held as (x y z 1), a quadratic as its 10 trailing coefficients.
__device__ void poly_lin_lin(const double a[4], const double b[4], double r[10]) {
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
__device__ void poly_quad_lin(const double a[10], const double b[4], double r[20]) {
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

// Francis double-shift QR (EISPACK hqr: exceptional shifts at 10 and 20 iterations, 30 n iterations in all) on the
// Hessenberg matrix a (eigenvalues only).  Called by the whole warp; wr/wi end up the same in every lane.
__device__ bool hessenberg_qr_warp(double (*a)[10], double wr[10], double wi[10], int lane) {
  const int n = 10;
  double anorm = 0;
  for (int i = 0; i < n; ++i) for (int j = i > 0 ? i - 1 : 0; j < n; ++j) anorm += fabs(a[i][j]);
  int nn = n - 1, itn = 30 * n;
  double t = 0;
  while (nn >= 0) {
    int its = 0, l;
    do {
      for (l = nn; l >= 1; --l) {
        double s = fabs(a[l - 1][l - 1]) + fabs(a[l][l]);
        if (s == 0.0) s = anorm;
        if (fabs(a[l][l - 1]) + s == s) break;
      }
      __syncwarp();
      if (l >= 1 && lane == 0) a[l][l - 1] = 0.0;
      __syncwarp();
      double x = a[nn][nn];
      if (l == nn) { wr[nn] = x + t; wi[nn] = 0.0; --nn; continue; }
      double y = a[nn - 1][nn - 1], w = a[nn][nn - 1] * a[nn - 1][nn];
      if (l == nn - 1) {
        const double p = 0.5 * (y - x), q = p * p + w;
        double z = sqrt(fabs(q));
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
      if (its == 10 || its == 20) {
        t += x;
        __syncwarp();
        if (lane <= nn) a[lane][lane] -= x;
        __syncwarp();
        const double s = fabs(a[nn][nn - 1]) + fabs(a[nn - 1][nn - 2]);
        y = x = 0.75 * s;
        w = -0.4375 * s * s;
      }
      ++its; --itn;
      int m;
      double p = 0, q = 0, r = 0, z;
      for (m = nn - 2; m >= l; --m) {
        z = a[m][m];
        r = x - z;
        double s = y - z;
        p = (r * s - w) / a[m + 1][m] + a[m][m + 1];
        q = a[m + 1][m + 1] - z - r - s;
        r = a[m + 2][m + 1];
        s = fabs(p) + fabs(q) + fabs(r);
        p /= s; q /= s; r /= s;
        if (m == l) break;
        const double u = fabs(a[m][m - 1]) * (fabs(q) + fabs(r));
        const double v = fabs(p) * (fabs(a[m - 1][m - 1]) + fabs(z) + fabs(a[m + 1][m + 1]));
        if (u + v == v) break;
      }
      __syncwarp();
      if (lane >= m + 2 && lane <= nn) { a[lane][lane - 2] = 0.0; if (lane != m + 2) a[lane][lane - 3] = 0.0; }
      __syncwarp();
      for (int k = m; k <= nn - 1; ++k) {
        if (k != m) {
          p = a[k][k - 1]; q = a[k + 1][k - 1]; r = 0.0;
          if (k != nn - 1) r = a[k + 2][k - 1];
          x = fabs(p) + fabs(q) + fabs(r);
          if (x != 0.0) { p /= x; q /= x; r /= x; }
        }
        const double sq = sqrt(p * p + q * q + r * r), s = p >= 0 ? sq : -sq;
        if (s == 0.0) continue;
        __syncwarp();
        if (lane == 0) {
          if (k == m) { if (l != m) a[k][k - 1] = -a[k][k - 1]; }
          else a[k][k - 1] = -s * x;
        }
        p += s; x = p / s; y = q / s; z = r / s; q /= p; r /= p;
        __syncwarp();
        if (lane >= k && lane <= nn) {             // rows k..k+2, one column per lane
          const int j = lane;
          double pp = a[k][j] + q * a[k + 1][j];
          if (k != nn - 1) { pp += r * a[k + 2][j]; a[k + 2][j] -= pp * z; }
          a[k + 1][j] -= pp * y; a[k][j] -= pp * x;
        }
        __syncwarp();
        const int mmin = nn < k + 3 ? nn : k + 3;
        if (lane >= l && lane <= mmin) {           // columns k..k+2, one row per lane
          const int i = lane;
          double pp = x * a[i][k] + y * a[i][k + 1];
          if (k != nn - 1) { pp += z * a[i][k + 2]; a[i][k + 2] -= pp * r; }
          a[i][k + 1] -= pp * q; a[i][k] -= pp;
        }
        __syncwarp();
      }
    } while (l < nn - 1);
  }
  return true;
}

// b1, b2: bearing vectors [.][3]; sample: the 5 indices.  Called by all 32 lanes of one warp; W.models / W.n_models out.
__device__ void five_point_warp(FivePointWork &W, const double *b1, const double *b2, const uint32_t *sample, int lane) {
  for (int e = lane; e < 81; e += 32) {                                   // A'A, EncodeEpipolarEquation rows
    const int i = e / 9, j = e % 9;
    double acc = 0;
    for (int t = 0; t < 5; ++t) {
      const size_t s = sample[t];
      acc += (b2[3 * s + i / 3] * b1[3 * s + i % 3]) * (b2[3 * s + j / 3] * b1[3 * s + j % 3]);
    }
    W.AtA[i][j] = acc;
    W.V[i][j] = i == j ? 1.0 : 0.0;
  }
  __syncwarp();
  double (*A)[9] = W.AtA, (*V)[9] = W.V;
  for (int sweep = 0; sweep < 60; ++sweep) {                              // cyclic Jacobi, the 9 k-updates over lanes
    double off = 0, diag = 0;
    for (int i = 0; i < 9; ++i) { diag += A[i][i] * A[i][i]; for (int j = i + 1; j < 9; ++j) off += A[i][j] * A[i][j]; }
    if (off <= 1e-60 * diag || off == 0.0) break;
    for (int p = 0; p < 8; ++p)
      for (int q = p + 1; q < 9; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        __syncwarp();
        if (lane < 9) { const int k = lane; const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
        __syncwarp();
        if (lane < 9) {
          const int k = lane;
          const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk;
          const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
        }
        __syncwarp();
      }
  }
  {                                                                        // the 4 smallest, ascending
    unsigned used = 0;
    for (int c = 0; c < 4; ++c) {
      int best = -1;
      for (int i = 0; i < 9; ++i) if (!(used >> i & 1u) && (best < 0 || A[i][i] < A[best][best])) best = i;
      used |= 1u << best;
      if (lane < 9) W.basis[lane][c] = V[lane][best];
    }
  }
  __syncwarp();
  const double (*E)[4] = W.basis;
  if (lane < 6) {                                                          // E E' (upper), one entry per lane
    const int P0[6] = {0, 0, 0, 1, 1, 2}, P1[6] = {0, 1, 2, 1, 2, 2};
    const int i = P0[lane], j = P1[lane];
    double t[10];
    poly_lin_lin(E[3 * i], E[3 * j], W.L[lane]);
    for (int k = 1; k < 3; ++k) { poly_lin_lin(E[3 * i + k], E[3 * j + k], t); for (int c = 0; c < 10; ++c) W.L[lane][c] += t[c]; }
  }
  __syncwarp();
  if (lane < 10) {
    const int c = lane;
    const double half_trace = 0.5 * (W.L[0][c] + W.L[3][c] + W.L[5][c]);
    W.L[0][c] -= half_trace; W.L[3][c] -= half_trace; W.L[5][c] -= half_trace;
  }
  __syncwarp();
  if (lane == 0) {                                                         // det E = 0
    const int T[3][4] = {{1, 5, 2, 4}, {2, 3, 0, 5}, {0, 4, 1, 3}};
    double *row = W.C[0];
    for (int c = 0; c < 20; ++c) row[c] = 0;
    for (int c = 0; c < 3; ++c) {
      double u[10], v[10], w[20];
      poly_lin_lin(E[T[c][0]], E[T[c][1]], u); poly_lin_lin(E[T[c][2]], E[T[c][3]], v);
      for (int k = 0; k < 10; ++k) u[k] -= v[k];
      poly_quad_lin(u, E[6 + c], w);
      for (int k = 0; k < 20; ++k) row[k] += w[k];
    }
  } else if (lane < 10) {                                                  // (E E' - tr/2) E = 0, one row per lane
    const int S3[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    const int i = (lane - 1) / 3, j = (lane - 1) % 3;
    double *row = W.C[lane], w[20];
    poly_quad_lin(W.L[S3[i][0]], E[j], row);
    for (int k = 1; k < 3; ++k) { poly_quad_lin(W.L[S3[i][k]], E[3 * k + j], w); for (int c = 0; c < 20; ++c) row[c] += w[c]; }
  }
  __syncwarp();
  double (*C)[20] = W.C;
  for (int k = 0; k < 10; ++k) {                                           // Gauss-Jordan, partial pivoting, one column per lane
    int piv = k;
    for (int r = k + 1; r < 10; ++r) if (fabs(C[r][k]) > fabs(C[piv][k])) piv = r;
    __syncwarp();
    if (piv != k && lane < 20) { const double a = C[k][lane]; C[k][lane] = C[piv][lane]; C[piv][lane] = a; }
    __syncwarp();
    if (lane < 10) W.f[lane] = lane == k ? 0.0 : C[lane][k] / C[k][k];
    __syncwarp();
    if (lane >= k && lane < 20) for (int r = 0; r < 10; ++r) if (r != k) C[r][lane] -= W.f[r] * C[k][lane];
    __syncwarp();
  }
  for (int e = lane; e < 100; e += 32) {                                   // the action matrix
    const int r = e / 10, c = e % 10;
    const int R[6] = {0, 1, 2, 4, 5, 7};
    double v = 0.0;
    if (r < 6) v = C[R[r]][10 + c] / C[R[r]][R[r]];
    else if ((r == 6 && c == 0) || (r == 7 && c == 1) || (r == 8 && c == 3) || (r == 9 && c == 6)) v = -1.0;
    W.At[r][c] = v; W.H[r][c] = v;
  }
  __syncwarp();
  double (*a)[10] = W.H;
  for (int m = 1; m < 9; ++m) {                                            // Householder reduction to Hessenberg form
    double scale = 0;
    for (int i = m; i < 10; ++i) scale += fabs(a[i][m - 1]);
    if (scale == 0.0) continue;
    double u[10], h = 0;
    for (int i = 9; i >= m; --i) { u[i] = a[i][m - 1] / scale; h += u[i] * u[i]; }
    const double g = u[m] > 0 ? -sqrt(h) : sqrt(h);
    h -= u[m] * g; u[m] -= g;
    if (lane >= m && lane < 10) {                                          // (I - u u'/h) A, one column per lane
      const int j = lane;
      double f = 0;
      for (int i = 9; i >= m; --i) f += u[i] * a[i][j];
      f /= h;
      for (int i = m; i < 10; ++i) a[i][j] -= f * u[i];
    }
    __syncwarp();
    if (lane < 10) {                                                       // A (I - u u'/h), one row per lane
      const int i = lane;
      double f = 0;
      for (int j = 9; j >= m; --j) f += u[j] * a[i][j];
      f /= h;
      for (int j = m; j < 10; ++j) a[i][j] -= f * u[j];
    }
    __syncwarp();
    if (lane == 0) { a[m][m - 1] = scale * g; for (int i = m + 1; i < 10; ++i) a[i][m - 1] = 0.0; }
    __syncwarp();
  }
  double wr[10], wi[10];
  const bool ok = hessenberg_qr_warp(a, wr, wi, lane);
  // one real eigenvalue per lane: null vector of At - lambda I (complete pivoting, last unknown = 1), E = basis * v[6..9]
  const bool real = ok && lane < 10 && wi[lane < 10 ? lane : 0] == 0.0;
  const unsigned bal = __ballot_sync(0xffffffffu, real);
  if (real) {
    const double lambda = wr[lane];
    double M[10][10], y[10], v[10]; int cp[10];
    for (int i = 0; i < 10; ++i) { cp[i] = i; for (int j = 0; j < 10; ++j) M[i][j] = W.At[i][j] - (i == j ? lambda : 0.0); }
    for (int k = 0; k < 9; ++k) {
      int pr = k, pc = k;
      for (int r = k; r < 10; ++r) for (int c = k; c < 10; ++c) if (fabs(M[r][c]) > fabs(M[pr][pc])) { pr = r; pc = c; }
      if (pr != k) for (int c = 0; c < 10; ++c) { const double tmp = M[k][c]; M[k][c] = M[pr][c]; M[pr][c] = tmp; }
      if (pc != k) { for (int r = 0; r < 10; ++r) { const double tmp = M[r][k]; M[r][k] = M[r][pc]; M[r][pc] = tmp; } const int ti = cp[k]; cp[k] = cp[pc]; cp[pc] = ti; }
      for (int r = k + 1; r < 10; ++r) {
        const double f = M[r][k] / M[k][k];
        for (int c = k; c < 10; ++c) M[r][c] -= f * M[k][c];
      }
    }
    y[9] = 1.0;
    for (int i = 8; i >= 0; --i) {
      double s = 0;
      for (int j = i + 1; j < 10; ++j) s += M[i][j] * y[j];
      y[i] = -s / M[i][i];
    }
    for (int i = 0; i < 10; ++i) v[cp[i]] = y[i];
    const int slot = __popc(bal & ((1u << lane) - 1u));
    for (int k = 0; k < 9; ++k) W.models[slot][k] = E[k][0] * v[6] + E[k][1] * v[7] + E[k][2] * v[8] + E[k][3] * v[9];
  }
  if (lane == 0) W.n_models = __popc(bal);
  __syncwarp();
}

// FundamentalFromEssential (multiview/essential.cpp:48-53): F = K_J^-T E K_I^-1
__device__ void fundamental_from_essential(const double *E, const double *intr, double *F) {
  const double KI[9] = {1.0 / intr[0], 0, -intr[1] / intr[0], 0, 1.0 / intr[0], -intr[2] / intr[0], 0, 0, 1.0};
  const double KJ[9] = {1.0 / intr[3], 0, -intr[4] / intr[3], 0, 1.0 / intr[3], -intr[5] / intr[3], 0, 0, 1.0};
  double T[9];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += KJ[3 * k + r] * E[3 * k + c]; T[3 * r + c] = v; }
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += T[3 * r + k] * KI[3 * k + c]; F[3 * r + c] = v; }
}

struct SmemE {                             // the essential instantiation's shared memory (Smem stays the F/H layout)
  uint32_t mt[624];
  FivePointWork fp;
  double Fm[10][9];                         // F in pixels of each real solution (E: fp.models)
  int hist[NBINS]; int n_le; int warp_cnt[THREADS / 32];
  uint32_t sample[7];
  int n_models, better_now;
  double nfa_thr, nfa_val;
};

// validation aid: one warp per sample of 5 bearing pairs
__global__ void __launch_bounds__(32) five_point_kernel(unsigned int n, const double *b1, const double *b2, double *E, int *n_models) {
  __shared__ FivePointWork W;
  __shared__ uint32_t sample[5];
  if (threadIdx.x < 5) sample[threadIdx.x] = threadIdx.x;
  __syncwarp();
  for (unsigned int s = blockIdx.x; s < n; s += gridDim.x) {
    five_point_warp(W, b1 + 15 * (size_t)s, b2 + 15 * (size_t)s, sample, threadIdx.x);
    for (int e = threadIdx.x; e < 90; e += 32) E[90 * (size_t)s + e] = e / 9 < W.n_models ? W.models[e / 9][e % 9] : 0.0;
    if (threadIdx.x == 0) n_models[s] = W.n_models;
    __syncwarp();
  }
}

// rand_sampling.hpp:35-58 / 71-95 (thread 0)
__device__ void sample_reject(Rng &g, int ms, uint32_t total, uint32_t *s) {
  int cnt = 0;
  while (cnt < ms) {
    const uint32_t v = lemire(g, total);
    bool found = false;
    for (int j = 0; j < cnt && !found; ++j) found = s[j] == v;
    if (!found) s[cnt++] = v;
  }
}
__device__ void sample_shuffle(Rng &g, int ms, uint32_t *vec_index, uint32_t size, uint32_t *s) {
  if ((uint32_t)ms > size) return;                             // UniformSample returns false and leaves the sample as it was
  const uint32_t last = size - 1;
  for (uint32_t i = 0; i < (uint32_t)ms; ++i) {
    const uint32_t k = i + lemire(g, last - i + 1);
    const uint32_t a = vec_index[i], b = vec_index[k]; vec_index[i] = b; vec_index[k] = a;
  }
  for (int i = 0; i < ms; ++i) s[i] = vec_index[i];
}

// ESSENTIAL = false: the F / H filter (A.model 0 / 1, normalised points, Smem); true: the E filter (five-point solver on
// bearing vectors, residuals in pixels against F = K_J^-T E K_I^-1, SmemE).
template <bool ESSENTIAL>
__global__ void __launch_bounds__(THREADS) acransac_kernel(Args A) {
  __shared__ typename std::conditional<ESSENTIAL, SmemE, Smem>::type S;
  const double INF = __longlong_as_double(0x7ff0000000000000ll);
  for (unsigned int pair = blockIdx.x; pair < A.n_pairs; pair += gridDim.x) {
    __syncthreads();
    const unsigned long long off = A.offsets[pair];
    const unsigned int nData = (unsigned int)(A.offsets[pair + 1] - off);
    const double *xI = A.xI + 2 * off, *xJ = A.xJ + 2 * off;
    double *x1 = A.x1 + (ESSENTIAL ? 3 : 2) * off, *x2 = A.x2 + (ESSENTIAL ? 3 : 2) * off;   // E: bearing vectors
    uint32_t *vec_index = A.vec_index + off, *inl = A.inliers + off;
    float *logc_n = A.logc_n + off + pair, *logc_k = A.logc_k + off + pair, *l10 = A.l10 + off + pair;
    if (threadIdx.x == 0) {
      A.n_inliers[pair] = 0; A.stats[2 * pair] = 0.0; A.stats[2 * pair + 1] = 0.0;
      for (int i = 0; i < 9; ++i) A.F[9 * (size_t)pair + i] = (i % 4 == 0) ? 1.0 : 0.0;
    }
    const int ms = ESSENTIAL ? 5 : A.model == 0 ? 7 : 4;           // MINIMUM_SAMPLES; MAX_MODELS = 10 / 3 / 1
    if (nData <= (unsigned int)ms) continue;                      // ACRANSAC: nData <= sizeSample -> {0, 0}
    // ---- kernel adaptor: normalisation (conditioning.cpp:54-77), logalpha0
    const int wI = A.image_size[4 * pair], hI = A.image_size[4 * pair + 1], wJ = A.image_size[4 * pair + 2], hJ = A.image_size[4 * pair + 3];
    double logalpha0, mult_error, maxThreshold;
    if constexpr (ESSENTIAL) {
      // ACKernelAdaptorEssential: no normalisation (N1 = N2 = I); bearings = normalize(K^-1 [x; 1]) (Camera_Pinhole.hpp:136-139)
      const double *k = A.intr + 6 * (size_t)pair;
      for (unsigned int i = threadIdx.x; i < nData; i += THREADS) {
        double u = (xI[2 * i] - k[1]) / k[0], v = (xI[2 * i + 1] - k[2]) / k[0], nrm = sqrt(u * u + v * v + 1.0);
        x1[3 * i] = u / nrm; x1[3 * i + 1] = v / nrm; x1[3 * i + 2] = 1.0 / nrm;
        u = (xJ[2 * i] - k[4]) / k[3]; v = (xJ[2 * i + 1] - k[5]) / k[3]; nrm = sqrt(u * u + v * v + 1.0);
        x2[3 * i] = u / nrm; x2[3 * i + 1] = v / nrm; x2[3 * i + 2] = 1.0 / nrm;
        vec_index[i] = i;
      }
      logalpha0 = log10(2. * hypot((double)wJ, (double)hJ) / (wJ * (double)hJ) / 0.5);
      mult_error = 0.5;
      maxThreshold = A.precision * A.precision;
    } else {
    if (threadIdx.x == 0) {
      const double d1 = 1.0 / sqrt((double)(wI * hI)), d2 = 1.0 / sqrt((double)(wJ * hJ));
      for (int i = 0; i < 9; ++i) { S.N1[i] = 0; S.N2[i] = 0; }
      S.N1[0] = S.N1[4] = d1; S.N1[8] = 1.0; S.N1[2] = (double)(-.5f * wI) * d1; S.N1[5] = -.5 * hI * d1;
      S.N2[0] = S.N2[4] = d2; S.N2[8] = 1.0; S.N2[2] = (double)(-.5f * wJ) * d2; S.N2[5] = -.5 * hJ * d2;
    }
    __syncthreads();
    for (unsigned int i = threadIdx.x; i < nData; i += THREADS) {
      x1[2 * i] = (S.N1[0] * xI[2 * i] + S.N1[2]) / 1.0; x1[2 * i + 1] = (S.N1[4] * xI[2 * i + 1] + S.N1[5]) / 1.0;
      x2[2 * i] = (S.N2[0] * xJ[2 * i] + S.N2[2]) / 1.0; x2[2 * i + 1] = (S.N2[4] * xJ[2 * i + 1] + S.N2[5]) / 1.0;
      vec_index[i] = i;
    }
    logalpha0 = A.model == 0 ? log10(2. * hypot((double)wJ, (double)hJ) / (wJ * (double)hJ) / S.N2[0])       // point to line
                             : log10(3.14159265358979323846 / (wJ * (double)hJ) / (S.N2[0] * S.N2[0]));   // point to point
    mult_error = A.model == 0 ? 0.5 : 1.0;
    maxThreshold = A.precision * A.precision * S.N2[0] * S.N2[0];
    }
    // ---- NFA tables (robust_estimator_ACRansac.hpp:57-119), float arithmetic in the reference's order
    for (unsigned int i = threadIdx.x; i <= nData; i += THREADS) l10[i] = (float)log10((double)(float)i);
    __syncthreads();
    for (unsigned int k = threadIdx.x; k <= nData; k += THREADS) {
      { unsigned int kk = k; float r = 0.f;                         // logcombi(k, n)
        if (kk < nData) { if (nData - kk < kk) kk = nData - kk; for (unsigned int i = 1; i <= kk; ++i) r += l10[nData - i + 1] - l10[i]; }
        logc_n[k] = r; }
      { unsigned int kk = (unsigned int)ms; const unsigned int m = k; float r = 0.f;   // logcombi(MINIMUM_SAMPLES, m)
        if (kk < m) { if (m - kk < kk) kk = m - kk; for (unsigned int i = 1; i <= kk; ++i) r += l10[m - i + 1] - l10[i]; }
        logc_k[k] = r; }
    }
    const double loge0 = log10((double)(ESSENTIAL ? 10 : A.model == 0 ? 3 : 1) * (double)(nData - ms));
    __syncthreads();
    // ---- ACRANSAC main loop (robust_estimator_ACRansac.hpp:330-480); the scalars live in every thread (uniform)
    Rng g{S.mt, 624};
    if (threadIdx.x == 0) rng_seed(g, 5489u);
    double minNFA = INF, errorMax = INF;
    int nIterReserve = (int)(A.iterations / 10);
    unsigned int nIter = A.iterations - nIterReserve;
    bool bACRansacMode = false;                                    // a finite precision is required (see the C entry point)
    unsigned int n_inl = 0, index_size = nData;
    for (unsigned int iter = 0; iter < nIter && iter < A.iterations; ++iter) {
      __syncthreads();
      if (threadIdx.x == 0) {
        if (bACRansacMode) sample_shuffle(g, ms, vec_index, index_size, S.sample); else sample_reject(g, ms, nData, S.sample);
      }
      __syncthreads();
      if constexpr (ESSENTIAL) {
        if (threadIdx.x < 32) {                                   // warp 0: the five-point solver, then F of each model
          five_point_warp(S.fp, x1, x2, S.sample, threadIdx.x);
          const int nm = S.fp.n_models;
          if (threadIdx.x < nm) fundamental_from_essential(S.fp.models[threadIdx.x], A.intr + 6 * (size_t)pair, S.Fm[threadIdx.x]);
          if (threadIdx.x == 0) S.n_models = nm;
        }
      } else {
      // A'A of the 7 epipolar constraints, summed in sample order
      if (threadIdx.x < 81) {
        const int i = threadIdx.x / 9, j = threadIdx.x % 9;
        double acc = 0;
        for (int t = 0; t < ms; ++t) {
          const unsigned int s = S.sample[t];
          const double x = x1[2 * s], y = x1[2 * s + 1], u = x2[2 * s], v = x2[2 * s + 1];
          if (A.model == 0) {                                     // EncodeEpipolarEquation (solver_fundamental_kernel.hpp:83-93)
            const double r[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
            acc += r[i] * r[j];
          } else {                                                // BuildActionMatrix (solver_homography_kernel.cpp:38-58): two rows per point
            const double r0[9] = {x, y, 1.0, 0, 0, 0, -u * x, -u * y, -u * 1.0};
            const double r1[9] = {0, 0, 0, x, y, 1.0, -v * x, -v * y, -v * 1.0};
            acc += r0[i] * r0[j] + r1[i] * r1[j];
          }
        }
        S.AtA[i][j] = acc;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        smallest_two_eigvecs(S.AtA, S.V, S.f1, S.f2);
        if (A.model != 0) { for (int t = 0; t < 9; ++t) S.models[0][t] = S.f1[t]; S.n_models = 1; }
        else {
        const double a = S.f1[0], j = S.f2[0], b = S.f1[1], k = S.f2[1], c = S.f1[2], l = S.f2[2], d = S.f1[3], m = S.f2[3], e = S.f1[4], n = S.f2[4],
                     f = S.f1[5], o = S.f2[5], gg = S.f1[6], p = S.f2[6], h = S.f1[7], q = S.f2[7], i = S.f1[8], r = S.f2[8];
        const double P[4] = {
          a*e*i + b*f*gg + c*d*h - a*f*h - b*d*i - c*e*gg,
          a*e*r + a*i*n + b*f*p + b*gg*o + c*d*q + c*h*m + d*h*l + e*i*j + f*gg*k -
          a*f*q - a*h*o - b*d*r - b*i*m - c*e*p - c*gg*n - d*i*k - e*gg*l - f*h*j,
          a*n*r + b*o*p + c*m*q + d*l*q + e*j*r + f*k*p + gg*k*o + h*l*m + i*j*n -
          a*o*q - b*m*r - c*n*p - d*k*r - e*l*p - f*j*q - gg*l*n - h*j*o - i*k*m,
          j*n*r + k*o*p + l*m*q - j*o*q - k*m*r - l*n*p};
        double roots[3]; int nr = 0;
        if (P[0] != 0.0) nr = solve_cubic(P[2] / P[3], P[1] / P[3], P[0] / P[3], roots);
        for (int kk = 0; kk < nr; ++kk) for (int t = 0; t < 9; ++t) S.models[kk][t] = S.f1[t] + roots[kk] * S.f2[t];
        S.n_models = nr;
        }
      }
      }
      __syncthreads();
      const int n_models = S.n_models;
      bool better = false;
      for (int mi = 0; mi < n_models; ++mi) {
        // residuals -> 20-bin histogram (histogram.hpp:65-77) and the max-consensus count
        if (threadIdx.x < NBINS) S.hist[threadIdx.x] = 0;
        if (threadIdx.x == 0) { S.n_le = 0; S.better_now = 0; }
        __syncthreads();
        const double by_interval = NBINS / (maxThreshold - 0.0);
        int le = 0;
        for (unsigned int i = threadIdx.x; i < nData; i += THREADS) {
          double e;
          if constexpr (ESSENTIAL) e = epipolar_error(S.Fm[mi], xI[2 * i], xI[2 * i + 1], xJ[2 * i], xJ[2 * i + 1]);
          else e = model_error(A.model, S.models[mi], x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
          if (e <= maxThreshold) ++le;
          if (e >= 0.0) { const unsigned long long b = (unsigned long long)((e - 0.0) * by_interval); if (b < (unsigned long long)NBINS) atomicAdd(&S.hist[(int)b], 1); }
        }
        if (!bACRansacMode) { for (int o = 16; o > 0; o >>= 1) le += __shfl_xor_sync(0xffffffffu, le, o); if ((threadIdx.x & 31) == 0) atomicAdd(&S.n_le, le); }
        __syncthreads();
        if (!bACRansacMode && (double)S.n_le > 2.5 * ms) bACRansacMode = true;       // (uniform: every thread reads the same count)
        if (bACRansacMode) {
          if (threadIdx.x == 0) {
            const double feps = (double)FLT_EPSILON;
            const double val = (maxThreshold - 0.0) / (double)(NBINS - 1);
            double best_nfa = INF, best_thr = 0.0;
            unsigned int cum = 0;
            for (int bin = 0; bin < NBINS; ++bin) {
              cum += (unsigned int)S.hist[bin];
              const double rv = val * (double)bin + 0.0;
              if (cum > (unsigned int)ms && rv > feps) {
                const double logalpha = logalpha0 + mult_error * log10(rv + feps);
                const double cur = loge0 + logalpha * (double)(cum - ms) + logc_n[cum] + logc_k[cum];
                if (cur < best_nfa && cur < 0) { best_nfa = cur; best_thr = rv; }
              }
            }
            if (best_nfa < minNFA) { S.better_now = 1; S.nfa_thr = best_thr; S.nfa_val = best_nfa; }
          }
          __syncthreads();
          if (S.better_now) {
            // inliers = { i : residual <= threshold } in ascending order (ordered block compaction)
            const double thr = S.nfa_thr;
            unsigned int base = 0;
            for (unsigned int i0 = 0; i0 < nData; i0 += THREADS) {
              const unsigned int i = i0 + threadIdx.x;
              bool in = false;
              if (i < nData) {
                if constexpr (ESSENTIAL) in = epipolar_error(S.Fm[mi], xI[2 * i], xI[2 * i + 1], xJ[2 * i], xJ[2 * i + 1]) <= thr;
                else in = model_error(A.model, S.models[mi], x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]) <= thr;
              }
              const unsigned int bal = __ballot_sync(0xffffffffu, in);
              if ((threadIdx.x & 31) == 0) S.warp_cnt[threadIdx.x >> 5] = __popc(bal);
              __syncthreads();
              unsigned int pre = base;
              for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pre += S.warp_cnt[w];
              if (in) inl[pre + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u))] = i;
              unsigned int tot = 0; for (int w = 0; w < THREADS / 32; ++w) tot += S.warp_cnt[w];
              base += tot;
              __syncthreads();
            }
            n_inl = base;
            // (the inlier list is overwritten even when the support is too small: ComputeNFA_and_inliers returns false
            //  then and the score is NOT updated, robust_estimator_ACRansac.hpp:243-256)
            if (n_inl > (unsigned int)ms) {
              better = true; minNFA = S.nfa_val; errorMax = thr;
              if (threadIdx.x < 9) {
                if constexpr (ESSENTIAL) A.F[9 * (size_t)pair + threadIdx.x] = S.fp.models[mi][threadIdx.x];
                else A.F[9 * (size_t)pair + threadIdx.x] = S.models[mi][threadIdx.x];
              }
            }
          }
        }
        __syncthreads();
      }
      if (!bACRansacMode && (int)iter > nIterReserve * 2) { nIter = 0; continue; }
      if (bACRansacMode && ((better && minNFA < 0) || ((iter + 1) == nIter && nIterReserve > 0))) {
        if (n_inl == 0) { ++nIter; --nIterReserve; }
        else {
          for (unsigned int i = threadIdx.x; i < n_inl; i += THREADS) vec_index[i] = inl[i];
          index_size = n_inl;
          if (nIterReserve) { nIter = iter + 1 + nIterReserve; nIterReserve = 0; }
        }
      }
    }
    __syncthreads();
    if (minNFA >= 0) n_inl = 0;
    if (threadIdx.x == 0) {
      A.n_inliers[pair] = n_inl;
      // E: Unnormalize does nothing and unormalizeError is the identity (errorMax stays squared)
      if constexpr (!ESSENTIAL) if (n_inl > 0) {
        double M[9], T[9], U[9];
        for (int i = 0; i < 9; ++i) M[i] = A.F[9 * (size_t)pair + i];
        if (A.model == 0) {      // UnnormalizerT: N2' * F * N1
          for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += S.N2[3 * k + r] * M[3 * k + c]; T[3 * r + c] = v; }
        } else {                 // UnnormalizerI: N2^-1 * H * N1
          const double d = S.N2[0], a2 = S.N2[2], b2 = S.N2[5];
          const double I2[9] = {1.0 / d, 0, -a2 / d, 0, 1.0 / d, -b2 / d, 0, 0, 1.0};
          for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += I2[3 * r + k] * M[3 * k + c]; T[3 * r + c] = v; }
        }
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double v = 0; for (int k = 0; k < 3; ++k) v += T[3 * r + k] * S.N1[3 * k + c]; U[3 * r + c] = v; }
        for (int i = 0; i < 9; ++i) A.F[9 * (size_t)pair + i] = U[i];
        errorMax = sqrt(errorMax) / S.N2[0];
      }
      A.stats[2 * pair] = errorMax; A.stats[2 * pair + 1] = minNFA;
    }
  }
}

// ---------------------------------------------------------------- angular essential models (DESIGN §3.10)
// GeometricFilter_ESphericalMatrix_AC_Angular<UPRIGHT> (matching_image_collection/E_ACRobust_Angular.hpp:52-160):
// ACKernelAdaptor_AngularRadianError<EightPointRelativePoseSolver | ThreePointUprightRelativePoseSolver, AngularError>
// + ACRANSAC on bearing vectors, then RelativePoseFromEssential on the AC-RANSAC inliers.  A sibling of
// acransac_kernel with its own arguments and shared memory, so the F/H and E instantiations are untouched.
struct AngArgs {
  const unsigned long long *offsets;       // [n_pairs + 1] into the match arrays
  const double *bI, *bJ;                   // [n_matches][3] bearing vectors of view I / J
  double max_threshold; unsigned int iterations;   // maxThreshold = D2R(precision) (squared radians), as ACRANSAC forms it
  float *logc_n, *logc_k, *l10;            // scratch [n_matches + n_pairs] each
  uint32_t *vec_index;                     // scratch [n_matches]
  uint32_t *inliers;                       // out [n_matches]: the first n_inliers[p] entries of pair p's segment
  uint32_t *n_inliers, *n_ransac;          // out [n_pairs]: after / before the cheirality step
  uint32_t *ransac_inliers;                // out [n_matches] or null: the AC-RANSAC list before the cheirality step
  double *E, *stats;                       // out [n_pairs][9], [n_pairs][2] = {errorMax (radians), minNFA}
  unsigned int n_pairs;
};

struct SmemAng {
  uint32_t mt[624];
  double AtA[9][9], V[9][9], f1[9], f2[9], model[9];
  double R[4][9], t[4][3];                 // the four poses of MotionFromEssential: rotation, translation()
  int hist[NBINS]; int n_le; int warp_cnt[THREADS / 32];
  int counts[4];
  uint32_t sample[8];
  int better_now, n_keep;
  double nfa_thr, nfa_val;
};

// AngularError::Error (solver_essential_eight_point.cpp:50-60): |asin(x2 . normalize(E x1))|, with the FMAs the
// reference's x86-64-v3 build forms (E x1: rows 0 and 1 as (E0 x0) + E1 x1 + E2 x2, row 2 as (E1 x1) + E2 x2 + E0 x0;
// the last term of the squared norm and of the dot product fused).  E row-major.
__device__ __forceinline__ double angular_error(const double *E, const double *a, const double *b) {
  double m0 = __fma_rn(E[2], a[2], __fma_rn(E[1], a[1], E[0] * a[0]));
  double m1 = __fma_rn(E[5], a[2], __fma_rn(E[4], a[1], E[3] * a[0]));
  double m2 = __fma_rn(E[6], a[0], __fma_rn(E[8], a[2], E[7] * a[1]));
  const double z = __fma_rn(m2, m2, m0 * m0 + m1 * m1);
  if (z > 0.0) { const double s = sqrt(z); m0 /= s; m1 /= s; m2 /= s; }
  return fabs(asin(__fma_rn(m2, b[2], b[0] * m0 + b[1] * m1)));
}

// cyclic Jacobi on a symmetric N x N (the same sweeps as smallest_two_eigvecs); A ends diagonal, V holds the vectors
template <int N>
__device__ void jacobi_sym(double (*A)[N], double (*V)[N]) {
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
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
        for (int k = 0; k < N; ++k) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk; }
        for (int k = 0; k < N; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq; }
      }
  }
}

// EightPointRelativePoseSolver::Solve (solver_essential_eight_point.cpp:15-46; the closest-essential projection runs
// only for more than 8 rows, never here) or ThreePointUprightRelativePoseSolver::Solve (solver_essential_three_point.cpp:
// 86-114).  A'A summed in sample order, one entry per thread; thread 0 runs Jacobi.  Called by the whole block; S.model out.
template <bool UPRIGHT>
__device__ void angular_solve(SmemAng &S, const double *b1, const double *b2, const uint32_t *sample) {
  if (UPRIGHT) {
    if (threadIdx.x < 16) {
      const int i = threadIdx.x / 4, j = threadIdx.x % 4;
      double acc = 0;
      for (int t = 0; t < 3; ++t) {
        const double *a = b1 + 3 * (size_t)sample[t], *b = b2 + 3 * (size_t)sample[t];
        const double r[4] = {a[0] * b[1], -a[2] * b[1], -b[0] * a[1], -b[2] * a[1]};
        acc += r[i] * r[j];
      }
      S.AtA[i][j] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double A4[4][4], V4[4][4];
      for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) A4[i][j] = S.AtA[i][j];
      jacobi_sym<4>(A4, V4);
      int k = 0; for (int i = 1; i < 4; ++i) if (A4[i][i] < A4[k][k]) k = i;
      for (int i = 0; i < 9; ++i) S.model[i] = 0.0;
      S.model[1] = V4[2][k]; S.model[3] = -V4[0][k]; S.model[5] = V4[1][k]; S.model[7] = V4[3][k];
    }
  } else {
    if (threadIdx.x < 81) {                                        // EncodeEpipolarEquation: row = x2(k) * x1'
      const int i = threadIdx.x / 9, j = threadIdx.x % 9;
      double acc = 0;
      for (int t = 0; t < 8; ++t) {
        const size_t s = sample[t];
        acc += (b2[3 * s + i / 3] * b1[3 * s + i % 3]) * (b2[3 * s + j / 3] * b1[3 * s + j % 3]);
      }
      S.AtA[i][j] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      smallest_two_eigvecs(S.AtA, S.V, S.f1, S.f2);
      for (int i = 0; i < 9; ++i) S.model[i] = S.f1[i];
    }
  }
  __syncthreads();
}

// MotionFromEssential (multiview/essential.cpp:79-113).  The SVD is formed from the Jacobi eigenvectors of E'E
// (descending): u_i = E v_i / |E v_i| for the two largest, u_3 = u_1 x u_2; then the reference's determinant fix-ups.
// Poses in the reference's order {(R0, t0), (R1, t1), (R0, t1), (R1, t0)}, each restated as Pose3(R, -R' t).translation().
__device__ void motion_from_essential(const double *E, double (*R)[9], double (*t)[3]) {
  double M[3][3], V[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double v = 0; for (int k = 0; k < 3; ++k) v += E[3 * k + i] * E[3 * k + j]; M[i][j] = v; }
  jacobi_sym<3>(M, V);
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a) for (int b = 0; b < 2 - a; ++b) if (M[o[b + 1]][o[b + 1]] > M[o[b]][o[b]]) { const int x = o[b]; o[b] = o[b + 1]; o[b + 1] = x; }
  double U[3][3], Vt[3][3];
  for (int c = 0; c < 3; ++c) for (int k = 0; k < 3; ++k) Vt[c][k] = V[k][o[c]];
  for (int c = 0; c < 2; ++c) {
    double u[3], n2 = 0;
    for (int r = 0; r < 3; ++r) { u[r] = E[3 * r] * Vt[c][0] + E[3 * r + 1] * Vt[c][1] + E[3 * r + 2] * Vt[c][2]; n2 += u[r] * u[r]; }
    const double n = sqrt(n2);
    for (int r = 0; r < 3; ++r) U[r][c] = u[r] / n;
  }
  U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
  U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
  U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
  auto det3 = [](const double (*m)[3]) {
    return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  };
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

// TriangulateIDWMidpoint (multiview/triangulation.cpp:179-216) between (I, 0) and (R, t): the Eq. (9) cheirality test
// only.  NaN norms (parallel rays) make every comparison false, as in the reference.
__device__ __forceinline__ bool idw_midpoint_cheirality(const double *R, const double *t, const double *x0, const double *x1) {
  double Rx0[3];
  for (int i = 0; i < 3; ++i) Rx0[i] = R[3 * i] * x0[0] + R[3 * i + 1] * x0[1] + R[3 * i + 2] * x0[2];
  auto norm_cross = [](const double *a, const double *b) {
    const double c0 = a[1] * b[2] - a[2] * b[1], c1 = a[2] * b[0] - a[0] * b[2], c2 = a[0] * b[1] - a[1] * b[0];
    return sqrt(c0 * c0 + c1 * c1 + c2 * c2);
  };
  const double p = norm_cross(Rx0, x1), q = norm_cross(Rx0, t), r = norm_cross(x1, t);
  const double l0 = r / p, l1 = q / p;
  double e[4] = {0, 0, 0, 0};                                      // t + l0 Rx0 -+ l1 x1, t - l0 Rx0 -+ l1 x1
  for (int i = 0; i < 3; ++i) {
    const double a = l0 * Rx0[i], b = l1 * x1[i];
    const double v0 = t[i] + a - b, v1 = t[i] + a + b, v2 = t[i] - a - b, v3 = t[i] - a + b;
    e[0] += v0 * v0; e[1] += v1 * v1; e[2] += v2 * v2; e[3] += v3 * v3;
  }
  // The reference takes std::min (vminsd), which fmin differs from only when an operand is NaN.  All four sums come from
  // the same l0, l1, t, Rx0, x1: a NaN in e[1..3] means a NaN l0 or l1, which makes e[0] NaN too, and then both forms
  // compare false.  With e[0] finite the two minima are equal.
  return e[0] < fmin(fmin(e[1], e[2]), e[3]);
}

// RelativePoseFromEssential (multiview/motion_from_essential.cpp:20-95) over idx[0..n), called by the whole block.  On
// true, idx[0..returned) is compacted in place to the chosen pose's list (ascending, as given); on false 0 is returned.
// S.counts holds the four cheirality counts afterwards.
__device__ unsigned int relative_pose_from_essential(SmemAng &S, const double *E, const double *b1, const double *b2,
                                                     uint32_t *idx, unsigned int n) {
  if (threadIdx.x == 0) motion_from_essential(E, S.R, S.t);
  if (threadIdx.x < 4) S.counts[threadIdx.x] = 0;
  __syncthreads();
  int c[4] = {0, 0, 0, 0};
  for (unsigned int k = threadIdx.x; k < n; k += THREADS) {
    const size_t i = idx[k];
    for (int p = 0; p < 4; ++p) c[p] += idw_midpoint_cheirality(S.R[p], S.t[p], b1 + 3 * i, b2 + 3 * i);
  }
  for (int p = 0; p < 4; ++p) {
    for (int o = 16; o > 0; o >>= 1) c[p] += __shfl_xor_sync(0xffffffffu, c[p], o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&S.counts[p], c[p]);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0; for (int p = 1; p < 4; ++p) if (S.counts[p] > S.counts[best]) best = p;   // the first maximal count
    int second = -1; for (int p = 0; p < 4; ++p) if (p != best && S.counts[p] > second) second = S.counts[p];
    const bool ok = S.counts[best] > 0 && second / (double)S.counts[best] < 0.7;
    S.n_keep = ok ? best : -1;
  }
  __syncthreads();
  const int best = S.n_keep;
  if (best < 0) return 0;
  unsigned int base = 0;
  for (unsigned int k0 = 0; k0 < n; k0 += THREADS) {                // ordered in-place compaction
    const unsigned int k = k0 + threadIdx.x;
    uint32_t i = 0; bool in = false;
    if (k < n) { i = idx[k]; in = idw_midpoint_cheirality(S.R[best], S.t[best], b1 + 3 * (size_t)i, b2 + 3 * (size_t)i); }
    const unsigned int bal = __ballot_sync(0xffffffffu, in);
    if ((threadIdx.x & 31) == 0) S.warp_cnt[threadIdx.x >> 5] = __popc(bal);
    __syncthreads();
    unsigned int pre = base;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pre += S.warp_cnt[w];
    if (in) idx[pre + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u))] = i;
    unsigned int tot = 0; for (int w = 0; w < THREADS / 32; ++w) tot += S.warp_cnt[w];
    base += tot;
    __syncthreads();
  }
  return base;
}

template <bool UPRIGHT>
__global__ void __launch_bounds__(THREADS) angular_acransac_kernel(AngArgs A) {
  __shared__ SmemAng S;
  const double INF = __longlong_as_double(0x7ff0000000000000ll);
  constexpr int ms = UPRIGHT ? 3 : 8;                             // MINIMUM_SAMPLES; MAX_MODELS = 1
  for (unsigned int pair = blockIdx.x; pair < A.n_pairs; pair += gridDim.x) {
    __syncthreads();
    const unsigned long long off = A.offsets[pair];
    const unsigned int nData = (unsigned int)(A.offsets[pair + 1] - off);
    const double *b1 = A.bI + 3 * off, *b2 = A.bJ + 3 * off;
    uint32_t *vec_index = A.vec_index + off, *inl = A.inliers + off;
    float *logc_n = A.logc_n + off + pair, *logc_k = A.logc_k + off + pair, *l10 = A.l10 + off + pair;
    if (threadIdx.x == 0) {
      A.n_inliers[pair] = 0; A.n_ransac[pair] = 0; A.stats[2 * pair] = 0.0; A.stats[2 * pair + 1] = 0.0;
      for (int i = 0; i < 9; ++i) A.E[9 * (size_t)pair + i] = (i % 4 == 0) ? 1.0 : 0.0;
    }
    if (nData <= (unsigned int)ms) continue;                      // ACRANSAC: {0, 0}; RelativePoseFromEssential on no inliers: false
    for (unsigned int i = threadIdx.x; i < nData; i += THREADS) vec_index[i] = i;
    // ACKernelAdaptor_AngularRadianError: no normalisation, logalpha0 = log10(1/2), multError = 1/4
    const double logalpha0 = log10(1. / 2.), mult_error = 1. / 4., maxThreshold = A.max_threshold;
    for (unsigned int i = threadIdx.x; i <= nData; i += THREADS) l10[i] = (float)log10((double)(float)i);
    __syncthreads();
    for (unsigned int k = threadIdx.x; k <= nData; k += THREADS) {
      { unsigned int kk = k; float r = 0.f;
        if (kk < nData) { if (nData - kk < kk) kk = nData - kk; for (unsigned int i = 1; i <= kk; ++i) r += l10[nData - i + 1] - l10[i]; }
        logc_n[k] = r; }
      { unsigned int kk = (unsigned int)ms; const unsigned int m = k; float r = 0.f;
        if (kk < m) { if (m - kk < kk) kk = m - kk; for (unsigned int i = 1; i <= kk; ++i) r += l10[m - i + 1] - l10[i]; }
        logc_k[k] = r; }
    }
    const double loge0 = log10((double)1 * (double)(nData - ms));
    __syncthreads();
    Rng g{S.mt, 624};
    if (threadIdx.x == 0) rng_seed(g, 5489u);
    double minNFA = INF, errorMax = INF;
    int nIterReserve = (int)(A.iterations / 10);
    unsigned int nIter = A.iterations - nIterReserve;
    bool bACRansacMode = false;
    unsigned int n_inl = 0, index_size = nData;
    for (unsigned int iter = 0; iter < nIter && iter < A.iterations; ++iter) {
      __syncthreads();
      if (threadIdx.x == 0) {
        if (bACRansacMode) sample_shuffle(g, ms, vec_index, index_size, S.sample); else sample_reject(g, ms, nData, S.sample);
      }
      __syncthreads();
      angular_solve<UPRIGHT>(S, b1, b2, S.sample);
      bool better = false;
      if (threadIdx.x < NBINS) S.hist[threadIdx.x] = 0;
      if (threadIdx.x == 0) { S.n_le = 0; S.better_now = 0; }
      __syncthreads();
      const double by_interval = NBINS / (maxThreshold - 0.0);
      int le = 0;
      for (unsigned int i = threadIdx.x; i < nData; i += THREADS) {
        const double a = angular_error(S.model, b1 + 3 * (size_t)i, b2 + 3 * (size_t)i), e = a * a;
        if (e <= maxThreshold) ++le;
        if (e >= 0.0) { const unsigned long long b = (unsigned long long)((e - 0.0) * by_interval); if (b < (unsigned long long)NBINS) atomicAdd(&S.hist[(int)b], 1); }
      }
      if (!bACRansacMode) { for (int o = 16; o > 0; o >>= 1) le += __shfl_xor_sync(0xffffffffu, le, o); if ((threadIdx.x & 31) == 0) atomicAdd(&S.n_le, le); }
      __syncthreads();
      if (!bACRansacMode && (double)S.n_le > 2.5 * ms) bACRansacMode = true;
      if (bACRansacMode) {
        if (threadIdx.x == 0) {
          const double feps = (double)FLT_EPSILON;
          const double val = (maxThreshold - 0.0) / (double)(NBINS - 1);
          double best_nfa = INF, best_thr = 0.0;
          unsigned int cum = 0;
          for (int bin = 0; bin < NBINS; ++bin) {
            cum += (unsigned int)S.hist[bin];
            const double rv = val * (double)bin + 0.0;
            if (cum > (unsigned int)ms && rv > feps) {
              const double logalpha = logalpha0 + mult_error * log10(rv + feps);
              const double cur = loge0 + logalpha * (double)(cum - ms) + logc_n[cum] + logc_k[cum];
              if (cur < best_nfa && cur < 0) { best_nfa = cur; best_thr = rv; }
            }
          }
          if (best_nfa < minNFA) { S.better_now = 1; S.nfa_thr = best_thr; S.nfa_val = best_nfa; }
        }
        __syncthreads();
        if (S.better_now) {
          const double thr = S.nfa_thr;
          unsigned int base = 0;
          for (unsigned int i0 = 0; i0 < nData; i0 += THREADS) {
            const unsigned int i = i0 + threadIdx.x;
            bool in = false;
            if (i < nData) { const double a = angular_error(S.model, b1 + 3 * (size_t)i, b2 + 3 * (size_t)i); in = a * a <= thr; }
            const unsigned int bal = __ballot_sync(0xffffffffu, in);
            if ((threadIdx.x & 31) == 0) S.warp_cnt[threadIdx.x >> 5] = __popc(bal);
            __syncthreads();
            unsigned int pre = base;
            for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pre += S.warp_cnt[w];
            if (in) inl[pre + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u))] = i;
            unsigned int tot = 0; for (int w = 0; w < THREADS / 32; ++w) tot += S.warp_cnt[w];
            base += tot;
            __syncthreads();
          }
          n_inl = base;
          if (n_inl > (unsigned int)ms) {
            better = true; minNFA = S.nfa_val; errorMax = thr;
            if (threadIdx.x < 9) A.E[9 * (size_t)pair + threadIdx.x] = S.model[threadIdx.x];
          }
        }
      }
      __syncthreads();
      if (!bACRansacMode && (int)iter > nIterReserve * 2) { nIter = 0; continue; }
      if (bACRansacMode && ((better && minNFA < 0) || ((iter + 1) == nIter && nIterReserve > 0))) {
        if (n_inl == 0) { ++nIter; --nIterReserve; }
        else {
          for (unsigned int i = threadIdx.x; i < n_inl; i += THREADS) vec_index[i] = inl[i];
          index_size = n_inl;
          if (nIterReserve) { nIter = iter + 1 + nIterReserve; nIterReserve = 0; }
        }
      }
    }
    __syncthreads();
    if (minNFA >= 0) n_inl = 0;
    if (threadIdx.x == 0) {
      A.n_ransac[pair] = n_inl;
      if (n_inl > 0) errorMax = sqrt(errorMax);                    // unormalizeError
      A.stats[2 * pair] = errorMax; A.stats[2 * pair + 1] = minNFA;
      for (int i = 0; i < 9; ++i) S.model[i] = A.E[9 * (size_t)pair + i];
    }
    if (A.ransac_inliers) for (unsigned int i = threadIdx.x; i < n_inl; i += THREADS) A.ransac_inliers[off + i] = inl[i];
    __syncthreads();
    const unsigned int n_final = relative_pose_from_essential(S, S.model, b1, b2, inl, n_inl);
    if (threadIdx.x == 0) A.n_inliers[pair] = n_final;
  }
}

// validation aids: one block per sample of ms bearing pairs / one RelativePoseFromEssential call
template <bool UPRIGHT>
__global__ void __launch_bounds__(THREADS) angular_solver_kernel(unsigned int n, const double *b1, const double *b2, double *E) {
  __shared__ SmemAng S;
  constexpr int ms = UPRIGHT ? 3 : 8;
  if (threadIdx.x < ms) S.sample[threadIdx.x] = threadIdx.x;
  for (unsigned int s = blockIdx.x; s < n; s += gridDim.x) {
    __syncthreads();
    angular_solve<UPRIGHT>(S, b1 + 3 * ms * (size_t)s, b2 + 3 * ms * (size_t)s, S.sample);
    if (threadIdx.x < 9) E[9 * (size_t)s + threadIdx.x] = S.model[threadIdx.x];
  }
}

__global__ void __launch_bounds__(THREADS) relative_pose_kernel(const double *E, const double *b1, const double *b2, uint32_t *idx,
                                                                unsigned int n, int *counts, unsigned int *n_out) {
  __shared__ SmemAng S;
  if (threadIdx.x < 9) S.model[threadIdx.x] = E[threadIdx.x];
  __syncthreads();
  const unsigned int k = relative_pose_from_essential(S, S.model, b1, b2, idx, n);
  if (threadIdx.x < 4) counts[threadIdx.x] = S.counts[threadIdx.x];
  if (threadIdx.x == 0) *n_out = k;                                // 0: false (true keeps at least the best count > 0)
}

}}  // namespace omvg::geom

namespace {

// everything after the per-model argument checks; intr (model OMVG_GEOM_ESSENTIAL only): [n_pairs][6]
int geom_run(int device, int32_t model, uint64_t n_pairs, const uint64_t *offsets, const double *xI, const double *xJ,
             const int32_t *image_size, const double *intr, double precision, uint32_t max_iterations,
             uint32_t *inliers, uint32_t *n_inliers, double *F, double *stats) {
  using namespace omvg;
  if (n_pairs && (!offsets || !image_size || !n_inliers || !F || !stats)) return fail(OMVG_E_ARG, "null argument");
  if (!(precision > 0.0) || !std::isfinite(precision)) return fail(OMVG_E_UNSUPPORTED, "the GPU filter needs a finite upper bound of the precision (main_GeometricFilter uses 4.0)");
  if (max_iterations < 1) return fail(OMVG_E_ARG, "max_iterations must be >= 1");
  int n_sms = 0;
  if (const int rc = check_device(device, &n_sms)) return rc;
  if (!n_pairs) return OMVG_OK;
  for (uint64_t p = 0; p < n_pairs; ++p) {
    if (offsets[p + 1] < offsets[p]) return fail(OMVG_E_ARG, "offsets must be non-decreasing");
    for (int k = 0; k < 4; ++k) if (image_size[4 * p + k] < 1 || image_size[4 * p + k] > 46340) return fail(OMVG_E_ARG, "pair %llu: bad image size", (unsigned long long)p);
  }
  const uint64_t nm = offsets[n_pairs];
  if (nm && (!xI || !xJ || !inliers)) return fail(OMVG_E_ARG, "null match arrays");
  if (nm >= (1ull << 31)) return fail(OMVG_E_UNSUPPORTED, "more than 2^31 putative matches in one call");
  const bool essential = model == OMVG_GEOM_ESSENTIAL;
  const size_t xs = essential ? 24 : 16;                  // scratch per match: bearing vectors (E) or normalised points
  OMVG_CUDA(cudaSetDevice(device));
  struct Call { cudaStream_t stream = nullptr; long long launches = 0; ~Call() { if (stream) cudaStreamDestroy(stream); } } call;
  OMVG_CUDA(cudaStreamCreateWithFlags(&call.stream, cudaStreamNonBlocking));
  const cudaStream_t st = call.stream;
  const size_t m1 = std::max<uint64_t>(nm, 1);            // no buffer is empty
  DevBuf<unsigned long long> d_off; DevBuf<double> d_xI, d_xJ, d_x1, d_x2, d_F, d_stats, d_intr; DevBuf<int> d_sz;
  DevBuf<float> d_ln, d_lk, d_l10; DevBuf<uint32_t> d_idx, d_inl, d_ninl;
  if (d_off.alloc(n_pairs + 1) || d_xI.alloc(2 * m1) || d_xJ.alloc(2 * m1) || d_x1.alloc(xs / 8 * m1) || d_x2.alloc(xs / 8 * m1) ||
      d_sz.alloc(4 * n_pairs) || d_ln.alloc(nm + n_pairs) || d_lk.alloc(nm + n_pairs) || d_l10.alloc(nm + n_pairs) ||
      d_idx.alloc(m1) || d_inl.alloc(m1) || d_ninl.alloc(n_pairs) || d_F.alloc(9 * n_pairs) || d_stats.alloc(2 * n_pairs) ||
      (essential && d_intr.alloc(6 * n_pairs)))
    return fail(OMVG_E_CUDA, "out of device memory");
  if (essential) OMVG_CUDA(cudaMemcpyAsync(d_intr.p, intr, n_pairs * 48, cudaMemcpyHostToDevice, st));
  OMVG_CUDA(cudaMemcpyAsync(d_off.p, offsets, (n_pairs + 1) * 8, cudaMemcpyHostToDevice, st));
  OMVG_CUDA(cudaMemcpyAsync(d_sz.p, image_size, n_pairs * 16, cudaMemcpyHostToDevice, st));
  if (nm) { OMVG_CUDA(cudaMemcpyAsync(d_xI.p, xI, nm * 16, cudaMemcpyHostToDevice, st)); OMVG_CUDA(cudaMemcpyAsync(d_xJ.p, xJ, nm * 16, cudaMemcpyHostToDevice, st)); }
  geom::Args A{};
  A.model = model;
  A.offsets = d_off.p; A.xI = d_xI.p; A.xJ = d_xJ.p; A.image_size = d_sz.p; A.precision = precision; A.iterations = max_iterations;
  A.x1 = d_x1.p; A.x2 = d_x2.p; A.logc_n = d_ln.p; A.logc_k = d_lk.p; A.l10 = d_l10.p; A.vec_index = d_idx.p; A.inliers = d_inl.p;
  A.n_inliers = d_ninl.p; A.F = d_F.p; A.stats = d_stats.p;
  A.n_pairs = (unsigned int)n_pairs; A.intr = d_intr.p;
  void (*kernel)(geom::Args) = essential ? geom::acransac_kernel<true> : geom::acransac_kernel<false>;
  int per_sm = 1; OMVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, geom::THREADS, 0));
  const unsigned int grid = (unsigned int)std::min<uint64_t>(n_pairs, (uint64_t)n_sms * std::max(1, per_sm));
  if (const int rc = launch(&call, kernel, grid, geom::THREADS, 0, A)) return rc;
  if (nm) OMVG_CUDA(cudaMemcpyAsync(inliers, d_inl.p, nm * 4, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaMemcpyAsync(n_inliers, d_ninl.p, n_pairs * 4, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaMemcpyAsync(F, d_F.p, n_pairs * 72, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaMemcpyAsync(stats, d_stats.p, n_pairs * 16, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaStreamSynchronize(st));
  return OMVG_OK;
}

}  // namespace

extern "C" int omvg_geom_acransac(int device, int32_t model, uint64_t n_pairs, const uint64_t *offsets, const double *xI, const double *xJ,
                                  const int32_t *image_size, double precision, uint32_t max_iterations,
                                  uint32_t *inliers, uint32_t *n_inliers, double *F, double *stats) {
  using namespace omvg;
  if (model != OMVG_GEOM_FUNDAMENTAL && model != OMVG_GEOM_HOMOGRAPHY) return fail(OMVG_E_UNSUPPORTED, "geometric model %d is not implemented on the GPU path (0 = fundamental, 1 = homography; the essential model needs intrinsics: omvg_geom_essential_acransac)", model);
  return geom_run(device, model, n_pairs, offsets, xI, xJ, image_size, nullptr, precision, max_iterations, inliers, n_inliers, F, stats);
}

extern "C" int omvg_geom_essential_acransac(int device, uint64_t n_pairs, const uint64_t *offsets, const double *xI, const double *xJ,
                                            const int32_t *image_size, const double *intr, double precision, uint32_t max_iterations,
                                            uint32_t *inliers, uint32_t *n_inliers, double *E, double *stats) {
  using namespace omvg;
  if (n_pairs && !intr) return fail(OMVG_E_ARG, "null intrinsics");
  for (uint64_t p = 0; p < n_pairs; ++p) {
    const double *k = intr + 6 * p;
    if (!(k[0] > 0.0) || !(k[3] > 0.0) || !std::isfinite(k[0]) || !std::isfinite(k[3])) return fail(OMVG_E_ARG, "pair %llu: the focal lengths must be finite and > 0", (unsigned long long)p);
    if (!std::isfinite(k[1]) || !std::isfinite(k[2]) || !std::isfinite(k[4]) || !std::isfinite(k[5])) return fail(OMVG_E_ARG, "pair %llu: non-finite principal point", (unsigned long long)p);
  }
  return geom_run(device, OMVG_GEOM_ESSENTIAL, n_pairs, offsets, xI, xJ, image_size, intr, precision, max_iterations, inliers, n_inliers, E, stats);
}

extern "C" int omvg_geom_debug_five_point(int device, uint32_t n, const double *b1, const double *b2, double *E, int32_t *n_models) {
  using namespace omvg;
  if (n && (!b1 || !b2 || !E || !n_models)) return fail(OMVG_E_ARG, "null argument");
  int n_sms = 0;
  if (const int rc = check_device(device, &n_sms)) return rc;
  if (!n) return OMVG_OK;
  OMVG_CUDA(cudaSetDevice(device));
  DevBuf<double, CudaAlloc> d_b1, d_b2, d_E; DevBuf<int, CudaAlloc> d_n;
  int rc;
  if ((rc = d_b1.alloc(15ull * n)) || (rc = d_b2.alloc(15ull * n)) || (rc = d_E.alloc(90ull * n)) || (rc = d_n.alloc(n))) return rc;
  OMVG_CUDA(cudaMemcpy(d_b1.p, b1, n * 120ull, cudaMemcpyHostToDevice)); OMVG_CUDA(cudaMemcpy(d_b2.p, b2, n * 120ull, cudaMemcpyHostToDevice));
  geom::five_point_kernel<<<std::min<uint32_t>(n, 64u * n_sms), 32>>>(n, d_b1.p, d_b2.p, d_E.p, d_n.p);
  OMVG_CUDA(cudaGetLastError());
  OMVG_CUDA(cudaMemcpy(E, d_E.p, n * 720ull, cudaMemcpyDeviceToHost)); OMVG_CUDA(cudaMemcpy(n_models, d_n.p, n * 4ull, cudaMemcpyDeviceToHost));
  return OMVG_OK;
}

namespace {

int check_bearings(const double *b, uint64_t n) {
  for (uint64_t i = 0; i < 3 * n; ++i) if (!std::isfinite(b[i])) return omvg::fail(OMVG_E_ARG, "non-finite bearing vector %llu", (unsigned long long)(i / 3));
  return OMVG_OK;
}

}  // namespace

extern "C" int omvg_geom_angular_acransac(int device, int32_t model, uint64_t n_pairs, const uint64_t *offsets,
                                          const double *bI, const double *bJ, double precision_deg, uint32_t max_iterations,
                                          uint32_t *inliers, uint32_t *n_inliers, double *E, double *stats, uint32_t *n_ransac_inliers,
                                          uint32_t *ransac_inliers) {
  using namespace omvg;
  if (model != OMVG_GEOM_ESSENTIAL_ANGULAR && model != OMVG_GEOM_ESSENTIAL_UPRIGHT) return fail(OMVG_E_ARG, "model %d is not an angular essential model (3 = eight-point, 4 = upright three-point)", model);
  if (n_pairs && (!offsets || !n_inliers || !E || !stats)) return fail(OMVG_E_ARG, "null argument");
  if (!(precision_deg > 0.0) || !std::isfinite(precision_deg)) return fail(OMVG_E_UNSUPPORTED, "the GPU filter needs a finite upper bound of the precision (main_GeometricFilter uses 4.0)");
  if (max_iterations < 1) return fail(OMVG_E_ARG, "max_iterations must be >= 1");
  int n_sms = 0;
  if (const int rc = check_device(device, &n_sms)) return rc;
  if (!n_pairs) return OMVG_OK;
  for (uint64_t p = 0; p < n_pairs; ++p) if (offsets[p + 1] < offsets[p]) return fail(OMVG_E_ARG, "offsets must be non-decreasing");
  const uint64_t nm = offsets[n_pairs];
  if (nm && (!bI || !bJ || !inliers)) return fail(OMVG_E_ARG, "null match arrays");
  if (nm >= (1ull << 31)) return fail(OMVG_E_UNSUPPORTED, "more than 2^31 putative matches in one call");
  if (const int rc = check_bearings(bI, nm)) return rc;
  if (const int rc = check_bearings(bJ, nm)) return rc;
  OMVG_CUDA(cudaSetDevice(device));
  struct Call { cudaStream_t stream = nullptr; long long launches = 0; ~Call() { if (stream) cudaStreamDestroy(stream); } } call;
  OMVG_CUDA(cudaStreamCreateWithFlags(&call.stream, cudaStreamNonBlocking));
  const cudaStream_t st = call.stream;
  const size_t m1 = std::max<uint64_t>(nm, 1);
  DevBuf<unsigned long long> d_off; DevBuf<double> d_bI, d_bJ, d_E, d_stats;
  DevBuf<float> d_ln, d_lk, d_l10; DevBuf<uint32_t> d_idx, d_inl, d_ninl, d_nr, d_rinl;
  if (d_off.alloc(n_pairs + 1) || d_bI.alloc(3 * m1) || d_bJ.alloc(3 * m1) || d_ln.alloc(nm + n_pairs) || d_lk.alloc(nm + n_pairs) ||
      d_l10.alloc(nm + n_pairs) || d_idx.alloc(m1) || d_inl.alloc(m1) || d_ninl.alloc(n_pairs) || d_nr.alloc(n_pairs) ||
      d_E.alloc(9 * n_pairs) || d_stats.alloc(2 * n_pairs) || (ransac_inliers && d_rinl.alloc(m1)))
    return fail(OMVG_E_CUDA, "out of device memory");
  OMVG_CUDA(cudaMemcpyAsync(d_off.p, offsets, (n_pairs + 1) * 8, cudaMemcpyHostToDevice, st));
  if (nm) { OMVG_CUDA(cudaMemcpyAsync(d_bI.p, bI, nm * 24, cudaMemcpyHostToDevice, st)); OMVG_CUDA(cudaMemcpyAsync(d_bJ.p, bJ, nm * 24, cudaMemcpyHostToDevice, st)); }
  geom::AngArgs A{};
  A.offsets = d_off.p; A.bI = d_bI.p; A.bJ = d_bJ.p;
  A.max_threshold = precision_deg * M_PI / 180.0;        // D2R (numeric.h:123-126); ACRANSAC takes it as the squared-error bound
  A.iterations = max_iterations;
  A.logc_n = d_ln.p; A.logc_k = d_lk.p; A.l10 = d_l10.p; A.vec_index = d_idx.p; A.inliers = d_inl.p;
  A.n_inliers = d_ninl.p; A.n_ransac = d_nr.p; A.ransac_inliers = ransac_inliers ? d_rinl.p : nullptr; A.E = d_E.p; A.stats = d_stats.p; A.n_pairs = (unsigned int)n_pairs;
  void (*kernel)(geom::AngArgs) = model == OMVG_GEOM_ESSENTIAL_UPRIGHT ? geom::angular_acransac_kernel<true> : geom::angular_acransac_kernel<false>;
  int per_sm = 1; OMVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, geom::THREADS, 0));
  const unsigned int grid = (unsigned int)std::min<uint64_t>(n_pairs, (uint64_t)n_sms * std::max(1, per_sm));
  if (const int rc = launch(&call, kernel, grid, geom::THREADS, 0, A)) return rc;
  if (nm) OMVG_CUDA(cudaMemcpyAsync(inliers, d_inl.p, nm * 4, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaMemcpyAsync(n_inliers, d_ninl.p, n_pairs * 4, cudaMemcpyDeviceToHost, st));
  if (n_ransac_inliers) OMVG_CUDA(cudaMemcpyAsync(n_ransac_inliers, d_nr.p, n_pairs * 4, cudaMemcpyDeviceToHost, st));
  if (ransac_inliers && nm) OMVG_CUDA(cudaMemcpyAsync(ransac_inliers, d_rinl.p, nm * 4, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaMemcpyAsync(E, d_E.p, n_pairs * 72, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaMemcpyAsync(stats, d_stats.p, n_pairs * 16, cudaMemcpyDeviceToHost, st));
  OMVG_CUDA(cudaStreamSynchronize(st));
  return OMVG_OK;
}

extern "C" int omvg_geom_debug_angular_solver(int device, int32_t model, uint32_t n, const double *b1, const double *b2, double *E) {
  using namespace omvg;
  if (model != OMVG_GEOM_ESSENTIAL_ANGULAR && model != OMVG_GEOM_ESSENTIAL_UPRIGHT) return fail(OMVG_E_ARG, "model %d is not an angular essential model", model);
  if (n && (!b1 || !b2 || !E)) return fail(OMVG_E_ARG, "null argument");
  int n_sms = 0;
  if (const int rc = check_device(device, &n_sms)) return rc;
  if (!n) return OMVG_OK;
  const size_t ms = model == OMVG_GEOM_ESSENTIAL_UPRIGHT ? 3 : 8;
  OMVG_CUDA(cudaSetDevice(device));
  DevBuf<double, CudaAlloc> d_b1, d_b2, d_E;
  int rc;
  if ((rc = d_b1.alloc(3 * ms * n)) || (rc = d_b2.alloc(3 * ms * n)) || (rc = d_E.alloc(9ull * n))) return rc;
  OMVG_CUDA(cudaMemcpy(d_b1.p, b1, 24 * ms * n, cudaMemcpyHostToDevice)); OMVG_CUDA(cudaMemcpy(d_b2.p, b2, 24 * ms * n, cudaMemcpyHostToDevice));
  const unsigned int grid = std::min<uint32_t>(n, 16u * n_sms);
  if (model == OMVG_GEOM_ESSENTIAL_UPRIGHT) geom::angular_solver_kernel<true><<<grid, geom::THREADS>>>(n, d_b1.p, d_b2.p, d_E.p);
  else geom::angular_solver_kernel<false><<<grid, geom::THREADS>>>(n, d_b1.p, d_b2.p, d_E.p);
  OMVG_CUDA(cudaGetLastError());
  OMVG_CUDA(cudaMemcpy(E, d_E.p, n * 72ull, cudaMemcpyDeviceToHost));
  return OMVG_OK;
}

extern "C" int omvg_geom_debug_relative_pose(int device, const double *E, uint32_t n_bearings, const double *b1, const double *b2,
                                             uint32_t n_index, const uint32_t *index, int32_t *counts, uint32_t *selected,
                                             uint32_t *n_selected, int32_t *result) {
  using namespace omvg;
  if (!E || !counts || !n_selected || !result || (n_bearings && (!b1 || !b2)) || (n_index && (!index || !selected))) return fail(OMVG_E_ARG, "null argument");
  for (int i = 0; i < 9; ++i) if (!std::isfinite(E[i])) return fail(OMVG_E_ARG, "non-finite E");
  for (uint32_t k = 0; k < n_index; ++k) if (index[k] >= n_bearings) return fail(OMVG_E_ARG, "index %u out of range", k);
  if (const int rc = check_bearings(b1, n_bearings)) return rc;
  if (const int rc = check_bearings(b2, n_bearings)) return rc;
  int n_sms = 0;
  if (const int rc = check_device(device, &n_sms)) return rc;
  OMVG_CUDA(cudaSetDevice(device));
  DevBuf<double, CudaAlloc> d_E, d_b1, d_b2; DevBuf<uint32_t, CudaAlloc> d_idx, d_n; DevBuf<int, CudaAlloc> d_c;
  int rc;
  if ((rc = d_E.alloc(9)) || (rc = d_b1.alloc(3ull * std::max(n_bearings, 1u))) || (rc = d_b2.alloc(3ull * std::max(n_bearings, 1u))) ||
      (rc = d_idx.alloc(std::max(n_index, 1u))) || (rc = d_n.alloc(1)) || (rc = d_c.alloc(4))) return rc;
  OMVG_CUDA(cudaMemcpy(d_E.p, E, 72, cudaMemcpyHostToDevice));
  if (n_bearings) { OMVG_CUDA(cudaMemcpy(d_b1.p, b1, 24ull * n_bearings, cudaMemcpyHostToDevice)); OMVG_CUDA(cudaMemcpy(d_b2.p, b2, 24ull * n_bearings, cudaMemcpyHostToDevice)); }
  if (n_index) OMVG_CUDA(cudaMemcpy(d_idx.p, index, 4ull * n_index, cudaMemcpyHostToDevice));
  geom::relative_pose_kernel<<<1, geom::THREADS>>>(d_E.p, d_b1.p, d_b2.p, d_idx.p, n_index, d_c.p, d_n.p);
  OMVG_CUDA(cudaGetLastError());
  OMVG_CUDA(cudaMemcpy(counts, d_c.p, 16, cudaMemcpyDeviceToHost));
  OMVG_CUDA(cudaMemcpy(n_selected, d_n.p, 4, cudaMemcpyDeviceToHost));
  if (*n_selected) OMVG_CUDA(cudaMemcpy(selected, d_idx.p, 4ull * *n_selected, cudaMemcpyDeviceToHost));
  *result = *n_selected > 0;
  return OMVG_OK;
}

extern "C" int omvg_geom_fundamental_acransac(int device, uint64_t n_pairs, const uint64_t *offsets, const double *xI, const double *xJ,
                                              const int32_t *image_size, double precision, uint32_t max_iterations,
                                              uint32_t *inliers, uint32_t *n_inliers, double *F, double *stats) {
  return omvg_geom_acransac(device, OMVG_GEOM_FUNDAMENTAL, n_pairs, offsets, xI, xJ, image_size, precision, max_iterations, inliers, n_inliers, F, stats);
}
