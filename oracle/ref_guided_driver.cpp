// ref_guided_driver.cpp — the reference's own guided matching behind a flat C ABI (checker of DESIGN §3.9).
//   ref_guided          ratio >= 0: geometry_aware::GuidedMatching<Mat3, Error>(model, camI, regionsI, camJ, regionsJ,
//                       thr, ratio, matches) on SIFT_Regions built from the arrays (guided_matching.hpp:178-227);
//                       ratio < 0: the descriptor-free GuidedMatching<Mat3, Error>(model, xI, xJ, thr, matches) on the
//                       positions PointsToMat would give (guided_matching.hpp:28-68)
//   ref_ud_pixels       IntrinsicBase::get_ud_pixel of a Pinhole_Intrinsic_Radial_K1
//   ref_guided_errors   EpipolarDistanceError::Error / AsymmetricError::Error
// Test infrastructure only; built by oracle/guided.mk into oracle/_ref.
#include "openMVG/cameras/Camera_Pinhole_Radial.hpp"
#include "openMVG/features/regions_factory.hpp"
#include "openMVG/multiview/solver_fundamental_kernel.hpp"
#include "openMVG/multiview/solver_homography_kernel.hpp"
#include "openMVG/robust_estimation/guided_matching.hpp"

#include <cstdint>
#include <memory>

using namespace openMVG;

namespace {

// cam6 = {w, h, f, ppx, ppy, k1} or nullptr
std::unique_ptr<cameras::IntrinsicBase> make_cam(const double *cam6) {
  if (!cam6) return nullptr;
  return std::unique_ptr<cameras::IntrinsicBase>(new cameras::Pinhole_Intrinsic_Radial_K1(
      (unsigned)cam6[0], (unsigned)cam6[1], cam6[2], cam6[3], cam6[4], cam6[5]));
}

std::unique_ptr<features::SIFT_Regions> make_regions(const double *xy, uint32_t n, const uint8_t *desc) {
  std::unique_ptr<features::SIFT_Regions> r(new features::SIFT_Regions);
  r->Features().resize(n); r->Descriptors().resize(n);
  for (uint32_t k = 0; k < n; ++k) {
    r->Features()[k] = features::SIOPointFeature(float(xy[2 * k]), float(xy[2 * k + 1]), 1.f, 0.f);
    for (int d = 0; d < 128; ++d) r->Descriptors()[k][d] = desc[128 * (size_t)k + d];
  }
  return r;
}

Mat positions(const cameras::IntrinsicBase * cam, const features::Regions & r) {
  Mat x(2, r.RegionCount());
  for (size_t k = 0; k < r.RegionCount(); ++k) x.col(k) = cam ? cam->get_ud_pixel(r.GetRegionPosition(k)) : r.GetRegionPosition(k);
  return x;
}

template <typename ErrorT>
void run(const Mat3 & M, const cameras::IntrinsicBase * camI, const features::Regions & rI, const cameras::IntrinsicBase * camJ,
         const features::Regions & rJ, double thr, double ratio, matching::IndMatches & m) {
  if (ratio >= 0) {
    geometry_aware::GuidedMatching<Mat3, ErrorT>(M, camI, rI, camJ, rJ, thr, ratio, m);
  } else {
    const Mat xI = positions(camI, rI), xJ = positions(camJ, rJ);
    geometry_aware::GuidedMatching<Mat3, ErrorT>(M, xI, xJ, thr, m);
  }
}

}  // namespace

extern "C" {

uint32_t ref_guided(int model, const double *xI, uint32_t nI, const uint8_t *dI, const double *xJ, uint32_t nJ, const uint8_t *dJ,
                    const double *M9, double thr, double ratio, const double *camI6, const double *camJ6, uint32_t *out_ij) {
  Mat3 M;
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M(r, c) = M9[3 * r + c];
  const auto camI = make_cam(camI6), camJ = make_cam(camJ6);
  const auto rI = make_regions(xI, nI, dI), rJ = make_regions(xJ, nJ, dJ);
  matching::IndMatches m;
  if (model == 0) run<fundamental::kernel::EpipolarDistanceError>(M, camI.get(), *rI, camJ.get(), *rJ, thr, ratio, m);
  else run<homography::kernel::AsymmetricError>(M, camI.get(), *rI, camJ.get(), *rJ, thr, ratio, m);
  for (size_t k = 0; k < m.size(); ++k) { out_ij[2 * k] = m[k].i_; out_ij[2 * k + 1] = m[k].j_; }
  return (uint32_t)m.size();
}

void ref_ud_pixels(const double *cam6, const double *xy, uint32_t n, double *out) {
  const auto cam = make_cam(cam6);
  for (uint32_t k = 0; k < n; ++k) {
    const Vec2 p = cam->get_ud_pixel(Vec2(xy[2 * k], xy[2 * k + 1]));
    out[2 * k] = p(0); out[2 * k + 1] = p(1);
  }
}

void ref_guided_errors(int model, const double *M9, const double *xI, const double *xJ, uint32_t n, double *err) {
  Mat3 M;
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M(r, c) = M9[3 * r + c];
  for (uint32_t k = 0; k < n; ++k) {
    const Vec2 x(xI[2 * k], xI[2 * k + 1]), y(xJ[2 * k], xJ[2 * k + 1]);
    err[k] = model == 0 ? fundamental::kernel::EpipolarDistanceError::Error(M, x, y) : homography::kernel::AsymmetricError::Error(M, x, y);
  }
}

}  // extern "C"
