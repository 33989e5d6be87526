// dropin_guided_test.cpp — guided matching exercised through openMVG's OWN types.
//
// TEST INFRASTRUCTURE ONLY.  Links the reference's compiled code (oracle/_ref objects) and libomvg_b200.so, then runs
// on one SfM_Data and one set of putative matches, for F (ratio 0.6), E (0.6), H (0.6) and H (-1: the descriptor-free variant)
//   reference  ImageCollectionGeometricFilter::Robust_model_estimation(GeometricFilter_?Matrix_AC(4.0, 2048), putative, true, ratio)
//   B200       ImageCollectionGeometricFilter_B200::Robust_model_estimation_?(putative, 4.0, 2048, nullptr, true, ratio)
// For H with ratio -1 the reference's own path cannot run: its PointsToMat (H_ACRobust.hpp:118-134) resizes the empty Mat
// it is given through an Eigen::Ref, which asserts in a debug build and writes through a null pointer otherwise.  The
// expectation there is composed from the reference's pieces as that code intends them: GeometricFilter_HMatrix_AC::
// Robust_estimation per pair, then GuidedMatching<Mat3, AsymmetricError>(m_H, xI, xJ, Square(m_dPrecision_robust)) on the
// 2 x n un-distorted positions, IndMatch::getDeduplicated and IndMatchDecorator<float>::getDeduplicated (:165-182).
// The scene has a Pinhole_Intrinsic_Radial_K1 view (positions get un-distorted), two different plain pinhole intrinsics,
// a view without an intrinsic, features at duplicated coordinates and a pair that fails the robust estimation.  The
// kept pairs and their guided matches must be identical.  Needs the GPU; run by tests/test_dropin_guided_gpu.py.
#include "openMVG/cameras/cameras.hpp"
#include "openMVG/features/regions_factory.hpp"
#include "openMVG/numeric/numeric.h"
#include "openMVG/sfm/sfm_data.hpp"
#include "openMVG/matching_image_collection/GeometricFilter.hpp"
#include "openMVG/matching_image_collection/E_ACRobust.hpp"
#include "openMVG/matching_image_collection/F_ACRobust.hpp"
#include "openMVG/matching_image_collection/H_ACRobust.hpp"

#include "openMVG/matching/indMatchDecoratorXY.hpp"
#include "openMVG/robust_estimation/guided_matching.hpp"

#include "../openmvg_b200/host/GeometricFilter_B200.hpp"

#include <algorithm>
#include <cstdio>
#include <memory>
#include <random>

using namespace openMVG;
using namespace openMVG::cameras;
using namespace openMVG::geometry;
using namespace openMVG::sfm;
using namespace openMVG::matching_image_collection;

namespace {

struct InMemory_Regions_Provider : public sfm::Regions_Provider
{
  void set(IndexT id, std::shared_ptr<features::Regions> r) { cache_[id] = std::move(r); }
  void set_type(features::Regions * r) { region_type_.reset(r); }
};

bool same(const matching::PairWiseMatches & A, const matching::PairWiseMatches & B, size_t & total)
{
  if (A.size() != B.size()) return false;
  total = 0;
  for (const auto & kv : A) {
    const auto it = B.find(kv.first);
    if (it == B.end() || it->second.size() != kv.second.size()) return false;
    for (size_t i = 0; i < kv.second.size(); ++i) if (kv.second[i].i_ != it->second[i].i_ || kv.second[i].j_ != it->second[i].j_) return false;
    total += kv.second.size();
  }
  return true;
}

// H with the descriptor-free guided step, from the reference's own pieces (see the header comment)
matching::PairWiseMatches reference_h_geometry_only(const SfM_Data & s, const std::shared_ptr<sfm::Regions_Provider> & provider,
                                                    const matching::PairWiseMatches & putative)
{
  matching::PairWiseMatches out;
  for (const auto & kv : putative) {
    GeometricFilter_HMatrix_AC f(4.0, 2048);
    matching::IndMatches inliers;
    if (!f.Robust_estimation(&s, provider, kv.first, kv.second, inliers)) continue;
    const IndexT ids[2] = {kv.first.first, kv.first.second};
    Mat x[2];
    features::PointFeatures feats[2];
    for (int k = 0; k < 2; ++k) {
      const View * v = s.views.at(ids[k]).get();
      const IntrinsicBase * cam = s.GetIntrinsics().count(v->id_intrinsic) ? s.GetIntrinsics().at(v->id_intrinsic).get() : nullptr;
      feats[k] = provider->get(ids[k])->GetRegionsPositions();
      x[k].resize(2, feats[k].size());
      for (size_t i = 0; i < feats[k].size(); ++i)
        x[k].col(i) = cam ? cam->get_ud_pixel({feats[k][i].x(), feats[k][i].y()}) : feats[k][i].coords().cast<double>();
    }
    matching::IndMatches m;
    geometry_aware::GuidedMatching<Mat3, homography::kernel::AsymmetricError>(f.m_H, x[0], x[1], Square(f.m_dPrecision_robust), m);
    matching::IndMatch::getDeduplicated(m);
    matching::IndMatchDecorator<float> deduplicator(m, feats[0], feats[1]);
    deduplicator.getDeduplicated(m);
    out.insert({kv.first, m});
  }
  return out;
}

}  // namespace

int main()
{
  std::setvbuf(stdout, nullptr, _IOLBF, 0);
  std::mt19937 g(29);
  std::uniform_real_distribution<double> U(-1.0, 1.0), U01(0.0, 1.0);
  std::normal_distribution<double> N(0, 1);
  SfM_Data s;
  s.intrinsics[0] = std::make_shared<Pinhole_Intrinsic_Radial_K1>(1600, 1200, 1700, 810, 590, 0.03);
  s.intrinsics[1] = std::make_shared<Pinhole_Intrinsic>(1600, 1200, 1500, 790, 610);
  s.intrinsics[2] = std::make_shared<Pinhole_Intrinsic>(1600, 1200, 1900, 805, 596);
  // view: 0 radial K1, 1 and 2 pinhole #1, 3 pinhole #2, 4 no intrinsic
  const IndexT view_intrinsic[5] = {0, 1, 1, 2, UndefinedIndexT};
  const int V = 5, P = 1200, D = 400, DUP = 25;                 // shared points, distractors, duplicated coordinates
  std::vector<Pose3> poses;
  for (int v = 0; v < V; ++v) {
    const Vec3 c(0.45 * v, 0.03 * v, 0.06 * v);
    const Vec3 aa(0.01 * v, -0.06 * v, 0.005 * v);
    const Mat3 R = aa.norm() > 0 ? Eigen::AngleAxisd(aa.norm(), aa.normalized()).toRotationMatrix() : Mat3(Mat3::Identity());
    poses.emplace_back(R, c);
    s.views[v] = std::make_shared<View>("", v, view_intrinsic[v], v, 1600, 1200);
  }
  auto provider = std::make_shared<InMemory_Regions_Provider>();
  provider->set_type(new features::SIFT_Regions);
  std::vector<Vec3> X(P);
  for (int j = 0; j < P; ++j) {                                 // 70 % on the plane z = 7 + 0.1 x, the rest in depth
    const double x = 1.6 * U(g), y = 1.2 * U(g);
    X[j] = Vec3(x, y, U01(g) < 0.7 ? 7.0 + 0.1 * x : 6.0 + 2.5 * U(g));
  }
  std::vector<std::array<int, 128>> base(P);
  for (auto & d : base) for (auto & c : d) c = int(U01(g) * 140);
  for (int v = 0; v < V; ++v) {
    // the view without an intrinsic still needs positions: project it with pinhole #1
    const IntrinsicBase * cam = s.intrinsics.at(v == 0 ? 0 : v == 3 ? 2 : 1).get();
    auto r = std::make_shared<features::SIFT_Regions>();
    r->Features().resize(P + D); r->Descriptors().resize(P + D);
    for (int j = 0; j < P + D; ++j) {
      Vec2 x;
      if (j < P) x = cam->project(poses[v](X[j])) + Vec2(0.4 * N(g), 0.4 * N(g));
      else x = Vec2(1600 * U01(g), 1200 * U01(g));
      r->Features()[j] = features::SIOPointFeature(float(x(0)), float(x(1)), 1.f, 0.f);
      for (int k = 0; k < 128; ++k) {
        const int val = j < P ? base[j][k] + int(9 * U01(g)) - 4 : int(U01(g) * 140);
        r->Descriptors()[j][k] = static_cast<unsigned char>(std::min(255, std::max(0, val)));
      }
    }
    for (int k = 0; k < DUP; ++k) r->Features()[P + k] = r->Features()[int(U01(g) * (P - 1))];   // duplicated coordinates
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
  bool fail = false;
  for (int run = 0; run < 4; ++run) {
    const char * name = run == 0 ? "F" : run == 1 ? "E" : "H";
    const double ratio = run == 3 ? -1.0 : 0.6;                 // main_GeometricFilter.cpp:284-320 passes -1 for H
    ImageCollectionGeometricFilter ref_filter(&s, base_provider);
    ImageCollectionGeometricFilter_B200 gpu_filter(&s, base_provider);
    matching::PairWiseMatches expected;
    bool ok = false;
    if (run == 0) {
      ref_filter.Robust_model_estimation(GeometricFilter_FMatrix_AC(4.0, 2048), putative, true, ratio);
      ok = gpu_filter.Robust_model_estimation_F(putative, 4.0, 2048, nullptr, true, ratio);
    } else if (run == 1) {
      ref_filter.Robust_model_estimation(GeometricFilter_EMatrix_AC(4.0, 2048), putative, true, ratio);
      ok = gpu_filter.Robust_model_estimation_E(putative, 4.0, 2048, nullptr, true, ratio);
    } else if (run == 2) {
      ref_filter.Robust_model_estimation(GeometricFilter_HMatrix_AC(4.0, 2048), putative, true, ratio);
      ok = gpu_filter.Robust_model_estimation_H(putative, 4.0, 2048, nullptr, true, ratio);
    } else {
      expected = reference_h_geometry_only(s, base_provider, putative);
      ok = gpu_filter.Robust_model_estimation_H(putative, 4.0, 2048, nullptr, true, ratio);
    }
    const auto & A = run == 3 ? expected : ref_filter.Get_geometric_matches();
    size_t total = 0;
    const bool identical = ok && same(A, gpu_filter.Get_geometric_matches(), total);
    const bool skipped_right = !A.count({1, 2}) && (run != 1 || std::none_of(A.begin(), A.end(), [](const std::pair<const Pair, matching::IndMatches> & kv) { return kv.first.second == 4; }));
    std::printf("GUIDED MATCHING (%s, ratio %g) drop-in: %zu of %zu pairs kept, %zu guided matches, %s\n", name, ratio, A.size(), putative.size(), total,
                identical ? "IDENTICAL" : "DIFFERENT");
    fail = fail || !identical || total == 0 || A.size() < 3 || !skipped_right;
  }
  std::printf(fail ? "DROPIN FAILED\n" : "DROPIN OK\n");
  return fail ? 1 : 0;
}
