// ref_geom_angular_driver.cpp — C entry points over the REFERENCE's own angular essential-matrix filters (test
// infrastructure only).  Compiled by oracle/angular.mk from $OPENMVG/src where it lies.  What
// GeometricFilter_ESphericalMatrix_AC_Angular<isUpright>::Robust_estimation (matching_image_collection/
// E_ACRobust_Angular.hpp:52-160) runs per image pair once the bearing vectors are formed:
//   ACKernelAdaptor_AngularRadianError<EightPointRelativePoseSolver | ThreePointUprightRelativePoseSolver, AngularError, Mat3>
//   ACRANSAC(kernel, inliers, iterations, &E, D2R(precision));
//   RelativePoseFromEssential(xI, xJ, E, inliers, &pose, &inliers_indexes, &X);
#include "openMVG/geometry/pose3.hpp"
#include "openMVG/multiview/essential.hpp"
#include "openMVG/multiview/motion_from_essential.hpp"
#include "openMVG/multiview/solver_essential_eight_point.hpp"
#include "openMVG/multiview/solver_essential_three_point.hpp"
#include "openMVG/multiview/triangulation.hpp"
#include "openMVG/numeric/numeric.h"
#include "openMVG/robust_estimation/robust_estimator_ACRansac.hpp"
#include "openMVG/robust_estimation/robust_estimator_ACRansacKernelAdaptator.hpp"

#include <cstdint>
#include <vector>

using namespace openMVG;
using namespace openMVG::robust;

namespace {

Mat3X to_mat(const double * b, int n) {
  Mat3X m(3, n);
  for (int i = 0; i < n; ++i) for (int c = 0; c < 3; ++c) m(c, i) = b[3 * i + c];
  return m;
}

// the cheirality count of each pose of MotionFromEssential, as RelativePoseFromEssential accumulates them
void cheirality_counts(const Mat3X & x1, const Mat3X & x2, const Mat3 & E, const std::vector<uint32_t> & idx, int32_t * counts) {
  std::vector<geometry::Pose3> poses;
  MotionFromEssential(E, &poses);
  const geometry::Pose3 pose1(Mat3::Identity(), Vec3::Zero());
  for (size_t p = 0; p < 4; ++p) {
    counts[p] = 0;
    Vec3 X;
    for (const uint32_t i : idx)
      if (Triangulate2View(pose1.rotation(), pose1.translation(), x1.col(i), poses[p].rotation(), poses[p].translation(), x2.col(i), X,
                           ETriangulationMethod::DEFAULT))
        ++counts[p];
  }
}

}  // namespace

extern "C" {

// model 3: EightPointRelativePoseSolver, 4: ThreePointUprightRelativePoseSolver, on n samples [n][ms][3]; E [n][9] row-major
void ref_angular_solver(int model, int n, const double * b1, const double * b2, double * E) {
  const int ms = model == 4 ? 3 : 8;
  for (int s = 0; s < n; ++s) {
    const Mat3X x1 = to_mat(b1 + 3 * ms * s, ms), x2 = to_mat(b2 + 3 * ms * s, ms);
    std::vector<Mat3> Es;
    if (model == 4) essential::kernel::ThreePointUprightRelativePoseSolver::Solve(x1, x2, &Es);
    else EightPointRelativePoseSolver::Solve(x1, x2, &Es);
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) E[9 * s + 3 * r + c] = Es.empty() ? 0.0 : Es[0](r, c);
  }
}

// AngularError::Error(E_k, b1_k, b2_k) for n candidates
void ref_angular_error(int n, const double * E, const double * b1, const double * b2, double * err) {
  for (int k = 0; k < n; ++k) {
    Mat3 M;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M(r, c) = E[9 * k + 3 * r + c];
    const Vec3 a(b1[3 * k], b1[3 * k + 1], b1[3 * k + 2]), b(b2[3 * k], b2[3 * k + 1], b2[3 * k + 2]);
    err[k] = AngularError::Error(M, a, b);
  }
}

// RelativePoseFromEssential(b1, b2, E, index): returns its boolean; counts[4], selected[*n_selected]
int ref_relative_pose(const double * E, int n_bearings, const double * b1, const double * b2, int n_index, const uint32_t * index,
                      int32_t * counts, uint32_t * selected, int32_t * n_selected) {
  const Mat3X x1 = to_mat(b1, n_bearings), x2 = to_mat(b2, n_bearings);
  Mat3 M;
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M(r, c) = E[3 * r + c];
  const std::vector<uint32_t> idx(index, index + n_index);
  cheirality_counts(x1, x2, M, idx, counts);
  geometry::Pose3 pose;
  std::vector<uint32_t> sel;
  std::vector<Vec3> X;
  const bool ok = RelativePoseFromEssential(x1, x2, M, idx, &pose, &sel, &X);
  *n_selected = ok ? (int32_t)sel.size() : 0;
  for (size_t k = 0; ok && k < sel.size(); ++k) selected[k] = sel[k];
  return ok;
}

// One pair of the filter on bearing vectors b1, b2 [n][3]; precision in degrees.  Returns the AC-RANSAC inlier count
// (ransac_inliers[n]); final_inliers[*n_final] is the list the functor keeps when it has more than 2.5 * ms entries;
// E[9] row-major, stats = {errorMax (radians), minNFA}, counts[4] the cheirality counts.
int ref_angular_acransac(int model, const double * b1, const double * b2, int n, double precision_deg, unsigned int iterations,
                         uint32_t * ransac_inliers, uint32_t * final_inliers, int32_t * n_final, double * E, double * stats, int32_t * counts) {
  const Mat3X x1 = to_mat(b1, n), x2 = to_mat(b2, n);
  Mat3 Em = Mat3::Identity();
  std::vector<uint32_t> vec_inliers;
  std::pair<double, double> out;
  if (model == 4) {
    using K = ACKernelAdaptor_AngularRadianError<essential::kernel::ThreePointUprightRelativePoseSolver, AngularError, Mat3>;
    const K kernel(x1, x2);
    out = ACRANSAC(kernel, vec_inliers, iterations, &Em, D2R(precision_deg));
  } else {
    using K = ACKernelAdaptor_AngularRadianError<EightPointRelativePoseSolver, AngularError, Mat3>;
    const K kernel(x1, x2);
    out = ACRANSAC(kernel, vec_inliers, iterations, &Em, D2R(precision_deg));
  }
  for (size_t i = 0; i < vec_inliers.size(); ++i) ransac_inliers[i] = vec_inliers[i];
  cheirality_counts(x1, x2, Em, vec_inliers, counts);
  geometry::Pose3 pose;
  std::vector<uint32_t> sel;
  std::vector<Vec3> X;
  const bool ok = RelativePoseFromEssential(x1, x2, Em, vec_inliers, &pose, &sel, &X);
  *n_final = ok ? (int32_t)sel.size() : 0;
  for (size_t k = 0; ok && k < sel.size(); ++k) final_inliers[k] = sel[k];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) E[3 * r + c] = Em(r, c);
  stats[0] = out.first; stats[1] = out.second;
  return (int)vec_inliers.size();
}

}  // extern "C"
