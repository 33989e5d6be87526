// dropin_angular_test.cpp — the angular essential-matrix geometric filters (`-g a`, `-g u`) exercised through openMVG's
// OWN types.
//
// TEST INFRASTRUCTURE ONLY.  Links the reference's compiled code (oracle/_ref objects) and libomvg_b200.so, then runs
// on one SfM_Data and one set of putative matches, for isUpright = false and true and with guided matching off and on,
//   reference  ImageCollectionGeometricFilter::Robust_model_estimation(GeometricFilter_ESphericalMatrix_AC_Angular<isUpright>(4.0, 2048),
//                                                                      putative, b_guided_matching)
//   B200       ImageCollectionGeometricFilter_B200::Robust_model_estimation_EAngular / _EUpright(putative, 4.0, 2048, nullptr,
//                                                                                               b_guided_matching)
// The scene has three spherical views (upright motion, points all around them, half behind), a Pinhole_Intrinsic_Radial_K1
// view (positions get un-distorted), two different plain pinhole intrinsics and a view without an intrinsic (its pairs
// are skipped).  Two pairs sit at the keep threshold: the reference keeps them with exactly 21 (eight-point) and 8
// (upright) matches; they are chosen by running the reference's functor on candidate match lists.  The kept pairs and
// their geometric matches must be identical.  Needs the GPU; run by tests/test_dropin_angular_gpu.py.
#include "openMVG/cameras/cameras.hpp"
#include "openMVG/features/regions_factory.hpp"
#include "openMVG/numeric/numeric.h"
#include "openMVG/sfm/sfm_data.hpp"
#include "openMVG/matching_image_collection/GeometricFilter.hpp"
#include "openMVG/matching_image_collection/E_ACRobust_Angular.hpp"

#include "../openmvg_b200/host/GeometricFilter_B200.hpp"

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

bool same_matches(const matching::PairWiseMatches & A, const matching::PairWiseMatches & B, size_t * total)
{
  *total = 0;
  if (A.size() != B.size()) return false;
  for (const auto & kv : A) {
    const auto it = B.find(kv.first);
    if (it == B.end() || it->second.size() != kv.second.size()) return false;
    for (size_t i = 0; i < kv.second.size(); ++i) if (kv.second[i].i_ != it->second[i].i_ || kv.second[i].j_ != it->second[i].j_) return false;
    *total += kv.second.size();
  }
  return true;
}

// a match list of n entries between views a and b over the points [0, n_points), `wrong` of them wrong correspondences
matching::IndMatches make_matches(std::mt19937 & g, int n, int n_points, double wrong)
{
  std::uniform_real_distribution<double> U01(0.0, 1.0);
  std::vector<int> js(n_points);
  for (int j = 0; j < n_points; ++j) js[j] = j;
  std::shuffle(js.begin(), js.end(), g);
  matching::IndMatches m;
  for (int k = 0; k < n; ++k) m.emplace_back(js[k], U01(g) < wrong ? int(U01(g) * (n_points - 1)) : js[k]);
  return m;
}

}  // namespace

int main()
{
  std::setvbuf(stdout, nullptr, _IOLBF, 0);
  std::mt19937 g(29);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  std::normal_distribution<double> N(0, 1);
  SfM_Data s;
  s.intrinsics[0] = std::make_shared<Intrinsic_Spherical>(2000, 1000);
  s.intrinsics[1] = std::make_shared<Pinhole_Intrinsic_Radial_K1>(1600, 1200, 1700, 810, 590, 0.03);
  s.intrinsics[2] = std::make_shared<Pinhole_Intrinsic>(1600, 1200, 1500, 790, 610);
  s.intrinsics[3] = std::make_shared<Pinhole_Intrinsic>(1600, 1200, 1900, 805, 596);
  // view: 0-2 spherical, 3 radial K1, 4 pinhole #1, 5 pinhole #2, 6 no intrinsic
  const IndexT view_intrinsic[7] = {0, 0, 0, 1, 2, 3, UndefinedIndexT};
  const int V = 7, P_FRONT = 900, P = 1300;                    // points [900, 1300) lie all around the spherical views
  std::vector<Pose3> poses;
  for (int v = 0; v < V; ++v) {
    Mat3 R; Vec3 c;
    if (v < 3) {                                                // upright: rotation about y, centre in the x-z plane
      R = Eigen::AngleAxisd(0.12 * v, Vec3::UnitY()).toRotationMatrix();
      c = Vec3(0.7 * v, 0.0, 0.25 * v);
    } else {
      const Vec3 aa(0.01 * v, -0.05 * v, 0.006 * v);
      R = Eigen::AngleAxisd(aa.norm(), aa.normalized()).toRotationMatrix();
      c = Vec3(0.3 * v, 0.03 * v, 0.05 * v);
    }
    poses.emplace_back(R, c);
    const IntrinsicBase * cam = s.intrinsics.at(v < 3 ? 0 : v == 3 ? 1 : v == 4 ? 2 : 3).get();
    s.views[v] = std::make_shared<View>("", v, view_intrinsic[v], v, cam->w(), cam->h());
  }
  auto provider = std::make_shared<InMemory_Regions_Provider>();
  provider->set_type(new features::SIFT_Regions);
  std::vector<Vec3> X(P);
  for (int j = 0; j < P_FRONT; ++j) X[j] = Vec3(1.5 * U(g), 1.1 * U(g), 7.0 + 2.0 * U(g));
  for (int j = P_FRONT; j < P; ++j) { const Vec3 d(N(g), N(g), N(g)); X[j] = d.normalized() * (4.0 + 3.0 * (1.0 + U(g))); }
  for (int v = 0; v < V; ++v) {
    // the view without an intrinsic still needs positions: project it with pinhole #2
    const IntrinsicBase * cam = s.intrinsics.at(v < 3 ? 0 : v == 3 ? 1 : v == 4 ? 2 : 3).get();
    auto r = std::make_shared<features::SIFT_Regions>();
    r->Features().resize(P); r->Descriptors().resize(P);
    const double noise = v < 3 ? 0.3 : 0.4;
    for (int j = 0; j < P; ++j) {
      const Vec2 x = cam->project(poses[v](X[j])) + Vec2(noise * N(g), noise * N(g));
      r->Features()[j] = features::SIOPointFeature(float(x(0)), float(x(1)), 1.f, 0.f);
    }
    provider->set(v, r);
  }
  const std::shared_ptr<sfm::Regions_Provider> base_provider = provider;

  // the two threshold pairs: the first candidate list the reference's functor keeps with exactly 21 / 8 matches
  matching::PairWiseMatches putative;
  const Pair thr_pair[2] = {{0, 1}, {1, 2}};
  const size_t thr_count[2] = {21, 8};
  for (int t = 0; t < 2; ++t) {
    bool found = false;
    for (int trial = 0; trial < 400 && !found; ++trial) {
      const matching::IndMatches m = make_matches(g, int(thr_count[t]) + 1 + trial % 4, P_FRONT, 0.1);
      matching::IndMatches kept;
      const bool ok = t == 0 ? GeometricFilter_ESphericalMatrix_AC_Angular<false>(4.0, 2048).Robust_estimation(&s, base_provider, thr_pair[t], m, kept)
                             : GeometricFilter_ESphericalMatrix_AC_Angular<true>(4.0, 2048).Robust_estimation(&s, base_provider, thr_pair[t], m, kept);
      if (ok && kept.size() == thr_count[t]) { putative.insert({thr_pair[t], m}); found = true; }
    }
    if (!found) { std::printf("no candidate list at the keep threshold for pair (%u, %u)\nDROPIN FAILED\n", thr_pair[t].first, thr_pair[t].second); return 1; }
  }
  for (int a = 0; a < V; ++a) for (int b = a + 1; b < V; ++b) {
    if (putative.count({a, b})) continue;
    const bool both_spherical = a < 3 && b < 3;
    putative.insert({{a, b}, make_matches(g, 250 + 40 * a + 10 * b, both_spherical ? P : P_FRONT, 0.35)});
  }

  bool fail = false;
  for (int upright = 0; upright < 2; ++upright) for (int guided = 0; guided < 2; ++guided) {
    ImageCollectionGeometricFilter ref_filter(&s, base_provider);
    if (upright) ref_filter.Robust_model_estimation(GeometricFilter_ESphericalMatrix_AC_Angular<true>(4.0, 2048), putative, guided != 0, 0.6);
    else ref_filter.Robust_model_estimation(GeometricFilter_ESphericalMatrix_AC_Angular<false>(4.0, 2048), putative, guided != 0, 0.6);
    ImageCollectionGeometricFilter_B200 gpu_filter(&s, base_provider);
    const bool ok = upright ? gpu_filter.Robust_model_estimation_EUpright(putative, 4.0, 2048, nullptr, guided != 0)
                            : gpu_filter.Robust_model_estimation_EAngular(putative, 4.0, 2048, nullptr, guided != 0);
    const auto & A = ref_filter.Get_geometric_matches(); const auto & B = gpu_filter.Get_geometric_matches();
    size_t total = 0;
    const bool same = ok && same_matches(A, B, &total);
    bool skipped_right = true, threshold_kept = false;
    for (const auto & kv : B) {
      if (kv.first.second == 6) skipped_right = false;            // view 6 has no intrinsic
      if (guided && !kv.second.empty()) skipped_right = false;     // -r: every kept pair holds the empty list
    }
    const auto th = A.find(thr_pair[upright]);
    if (guided) threshold_kept = th != A.end();
    else threshold_kept = th != A.end() && th->second.size() == thr_count[upright];
    std::printf("GEOMETRIC FILTER (%s, -r %s) drop-in: %zu of %zu pairs kept, %zu geometric matches, threshold pair (%u, %u) %s, %s\n",
                upright ? "upright E, -g u" : "angular E, -g a", guided ? "on" : "off", A.size(), putative.size(), total,
                thr_pair[upright].first, thr_pair[upright].second, threshold_kept ? "kept" : "NOT KEPT", same ? "IDENTICAL" : "DIFFERENT");
    if (!same || A.size() < 6 || !skipped_right || !threshold_kept || (!guided && total == 0)) fail = true;
  }
  std::printf(fail ? "DROPIN FAILED\n" : "DROPIN OK\n");
  return fail ? 1 : 0;
}
