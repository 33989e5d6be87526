// dropin_essential_test.cpp — the essential-matrix geometric filter exercised through openMVG's OWN types.
//
// TEST INFRASTRUCTURE ONLY.  Links the reference's compiled code (oracle/_ref objects) and libomvg_b200.so, then runs
// on one SfM_Data and one set of putative matches
//   reference  ImageCollectionGeometricFilter::Robust_model_estimation(GeometricFilter_EMatrix_AC(4.0, 2048), putative)
//   B200       ImageCollectionGeometricFilter_B200::Robust_model_estimation_E(putative, 4.0, 2048)
// The scene has a Pinhole_Intrinsic_Radial_K1 view (positions get un-distorted), two different plain pinhole intrinsics,
// a view without an intrinsic and a spherical view (both filters skip the pairs that touch them), and a pair with too few
// matches.  The kept pairs and their geometric matches must be identical.  Needs the GPU; run by
// tests/test_dropin_essential_gpu.py.
#include "openMVG/cameras/cameras.hpp"
#include "openMVG/features/regions_factory.hpp"
#include "openMVG/numeric/numeric.h"
#include "openMVG/sfm/sfm_data.hpp"
#include "openMVG/matching_image_collection/GeometricFilter.hpp"
#include "openMVG/matching_image_collection/E_ACRobust.hpp"

#include "../openmvg_b200/host/GeometricFilter_B200.hpp"

#include <cstdio>
#include <memory>
#include <random>

using namespace openMVG;
using namespace openMVG::cameras;
using namespace openMVG::geometry;
using namespace openMVG::sfm;

namespace {

struct InMemory_Regions_Provider : public sfm::Regions_Provider
{
  void set(IndexT id, std::shared_ptr<features::Regions> r) { cache_[id] = std::move(r); }
  void set_type(features::Regions * r) { region_type_.reset(r); }
};

}  // namespace

int main()
{
  std::setvbuf(stdout, nullptr, _IOLBF, 0);
  std::mt19937 g(23);
  std::uniform_real_distribution<double> U(-1.0, 1.0), U01(0.0, 1.0);
  std::normal_distribution<double> N(0, 1);
  SfM_Data s;
  s.intrinsics[0] = std::make_shared<Pinhole_Intrinsic_Radial_K1>(1600, 1200, 1700, 810, 590, 0.03);
  s.intrinsics[1] = std::make_shared<Pinhole_Intrinsic>(1600, 1200, 1500, 790, 610);
  s.intrinsics[2] = std::make_shared<Pinhole_Intrinsic>(1600, 1200, 1900, 805, 596);
  s.intrinsics[3] = std::make_shared<Intrinsic_Spherical>(1600, 1200);
  // view: 0 radial K1, 1 and 2 pinhole #1, 3 pinhole #2, 4 no intrinsic, 5 spherical
  const IndexT view_intrinsic[6] = {0, 1, 1, 2, UndefinedIndexT, 3};
  const int V = 6, P = 900;
  std::vector<Pose3> poses;
  for (int v = 0; v < V; ++v) {
    const Vec3 c(0.5 * v, 0.04 * v, 0.08 * v);
    const Vec3 aa(0.01 * v, -0.07 * v, 0.006 * v);
    const Mat3 R = aa.norm() > 0 ? Eigen::AngleAxisd(aa.norm(), aa.normalized()).toRotationMatrix() : Mat3(Mat3::Identity());
    poses.emplace_back(R, c);
    s.views[v] = std::make_shared<View>("", v, view_intrinsic[v], v, 1600, 1200);
  }
  auto provider = std::make_shared<InMemory_Regions_Provider>();
  provider->set_type(new features::SIFT_Regions);
  std::vector<Vec3> X(P);
  for (auto & x : X) x = Vec3(1.5 * U(g), 1.2 * U(g), 6.5 + 2.5 * U(g));
  for (int v = 0; v < V; ++v) {
    // the views without a pinhole intrinsic still need positions: project them with pinhole #1
    const IntrinsicBase * cam = s.intrinsics.at(v == 0 ? 0 : v == 3 ? 2 : 1).get();
    auto r = std::make_shared<features::SIFT_Regions>();
    r->Features().resize(P); r->Descriptors().resize(P);
    for (int j = 0; j < P; ++j) {
      const Vec2 x = cam->project(poses[v](X[j])) + Vec2(0.4 * N(g), 0.4 * N(g));
      r->Features()[j] = features::SIOPointFeature(float(x(0)), float(x(1)), 1.f, 0.f);
    }
    provider->set(v, r);
  }
  matching::PairWiseMatches putative;
  for (int a = 0; a < V; ++a) for (int b = a + 1; b < V; ++b) {
    matching::IndMatches m;
    const int n = (a == 1 && b == 2) ? 12 : 300 + 100 * a;                                 // one pair with too few matches
    for (int j = 0; j < n; ++j) m.emplace_back(j, U01(g) < 0.35 ? int(U01(g) * (P - 1)) : j);   // 35 % wrong correspondences
    putative.insert({{a, b}, m});
  }
  const std::shared_ptr<sfm::Regions_Provider> base_provider = provider;
  matching_image_collection::ImageCollectionGeometricFilter ref_filter(&s, base_provider);
  ref_filter.Robust_model_estimation(matching_image_collection::GeometricFilter_EMatrix_AC(4.0, 2048), putative);
  matching_image_collection::ImageCollectionGeometricFilter_B200 gpu_filter(&s, base_provider);
  const bool ok = gpu_filter.Robust_model_estimation_E(putative, 4.0, 2048);
  const auto & A = ref_filter.Get_geometric_matches(); const auto & B = gpu_filter.Get_geometric_matches();
  bool same = ok && A.size() == B.size();
  size_t total = 0;
  for (const auto & kv : A) {
    const auto it = B.find(kv.first);
    if (it == B.end() || it->second.size() != kv.second.size()) { same = false; break; }
    for (size_t i = 0; i < kv.second.size(); ++i) if (kv.second[i].i_ != it->second[i].i_ || kv.second[i].j_ != it->second[i].j_) { same = false; break; }
    total += kv.second.size();
  }
  // pairs among views 0-3 only can be kept, and (1, 2) has too few matches: at most 5 of the 15
  bool skipped_right = true;
  for (const auto & kv : B) if (kv.first.first > 3 || kv.first.second > 3 || (kv.first.first == 1 && kv.first.second == 2)) skipped_right = false;
  std::printf("GEOMETRIC FILTER (E, AC-RANSAC) drop-in: %zu of %zu pairs kept, %zu geometric matches, %s\n", A.size(), putative.size(), total,
              same ? "IDENTICAL" : "DIFFERENT");
  const bool fail = !same || total == 0 || A.size() < 4 || !skipped_right;
  std::printf(fail ? "DROPIN FAILED\n" : "DROPIN OK\n");
  return fail ? 1 : 0;
}
