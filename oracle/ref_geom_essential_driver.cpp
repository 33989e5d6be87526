// ref_geom_essential_driver.cpp — C entry points over the REFERENCE's own essential-matrix filter (test infrastructure
// only).  Compiled by oracle/essential.mk from $OPENMVG/src where it lies.  What GeometricFilter_EMatrix_AC::
// Robust_estimation (matching_image_collection/E_ACRobust.hpp:55-150) runs per image pair after MatchesPairToMat:
//   ACKernelAdaptorEssential<FivePointSolver, EpipolarDistanceError, Mat3> kernel(xI, (*cam_I)(xI), wI, hI,
//                                                                              xJ, (*cam_J)(xJ), wJ, hJ, K_I, K_J);
//   ACRANSAC(kernel, inliers, iterations, &E, Square(precision));
#include "openMVG/cameras/Camera_Pinhole.hpp"
#include "openMVG/multiview/solver_essential_five_point.hpp"
#include "openMVG/multiview/solver_essential_kernel.hpp"
#include "openMVG/multiview/solver_fundamental_kernel.hpp"
#include "openMVG/numeric/numeric.h"
#include "openMVG/robust_estimation/robust_estimator_ACRansac.hpp"
#include "openMVG/robust_estimation/robust_estimator_ACRansacKernelAdaptator.hpp"

#include <cstdint>
#include <vector>

using namespace openMVG;
using namespace openMVG::robust;

extern "C" {

// FivePointsRelativePose on n samples of 5 bearing pairs ([n][5][3] each).  E: [n][10][9] row-major, n_models[n].
void ref_five_point(int n, const double * b1, const double * b2, double * E, int32_t * n_models)
{
  for (int s = 0; s < n; ++s) {
    Mat3X x1(3, 5), x2(3, 5);
    for (int t = 0; t < 5; ++t) for (int c = 0; c < 3; ++c) { x1(c, t) = b1[15 * s + 3 * t + c]; x2(c, t) = b2[15 * s + 3 * t + c]; }
    std::vector<Mat3> Es;
    FivePointsRelativePose(x1, x2, &Es);
    n_models[s] = (int32_t)Es.size();
    for (size_t m = 0; m < Es.size() && m < 10; ++m)
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) E[90 * s + 9 * m + 3 * r + c] = Es[m](r, c);
  }
}

// xI, xJ: n pixel positions each, interleaved (x, y).  intr = {f, ppx, ppy} of view I then view J.  precision: upper
// bound in pixels.  Returns the number of inliers (> 2.5 * 5 for the pair to be kept).  out: inliers[n] (ascending),
// E[9] row-major, stats = {errorMax (squared pixels: unormalizeError is the identity), minNFA}.
int ref_acransac_essential(const double * xI, const double * xJ, int n, int wI, int hI, int wJ, int hJ, const double * intr,
                           double precision, unsigned int iterations, uint32_t * inliers, double * E, double * stats)
{
  Mat2X a(2, n), b(2, n);
  for (int i = 0; i < n; ++i) { a(0, i) = xI[2 * i]; a(1, i) = xI[2 * i + 1]; b(0, i) = xJ[2 * i]; b(1, i) = xJ[2 * i + 1]; }
  const cameras::Pinhole_Intrinsic camI(wI, hI, intr[0], intr[1], intr[2]), camJ(wJ, hJ, intr[3], intr[4], intr[5]);
  using KernelType = ACKernelAdaptorEssential<essential::kernel::FivePointSolver, fundamental::kernel::EpipolarDistanceError, Mat3>;
  const KernelType kernel(a, camI(a), wI, hI, b, camJ(b), wJ, hJ, camI.K(), camJ.K());
  Mat3 Em = Mat3::Identity();
  std::vector<uint32_t> vec_inliers;
  const std::pair<double, double> out = ACRANSAC(kernel, vec_inliers, iterations, &Em, Square(precision));
  for (size_t i = 0; i < vec_inliers.size(); ++i) inliers[i] = vec_inliers[i];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) E[3 * r + c] = Em(r, c);
  stats[0] = out.first; stats[1] = out.second;
  return (int)vec_inliers.size();
}

}  // extern "C"
