// ImageCollectionGeometricFilter_B200 — the fundamental-matrix geometric filter of openMVG_main_GeometricFilter on the
// B200: drop-in for
//     ImageCollectionGeometricFilter(sfm_data, regions_provider)
//       .Robust_model_estimation(GeometricFilter_FMatrix_AC(dPrecision, iteration), putative_matches[, b_guided_matching, d_distance_ratio])
// (reference: matching_image_collection/GeometricFilter.hpp:44-133, F_ACRobust.hpp:45-106, called at
// software/SfM/main_GeometricFilter.cpp:300-308).  The per-pair feature positions come from openMVG's own
// MatchesPairToMat (un-distorted when the view has an intrinsic), all pairs go to the device in ONE call of
// omvg_geom_fundamental_acransac (one CTA per pair; same MT19937 sample sequence and NFA decisions as ACRANSAC), and a
// pair is kept iff it has more than 2.5 * 7 inliers (F_ACRobust.hpp:85).
//
// Robust_model_estimation_H is the same for GeometricFilter_HMatrix_AC (H_ACRobust.hpp: 4-point homography).
// Robust_model_estimation_E is GeometricFilter_EMatrix_AC (E_ACRobust.hpp:55-150: five-point essential matrix of calibrated
// views): pairs whose views lack an intrinsic or have a non-pinhole one are skipped and not kept, as the reference skips
// them; K comes from Pinhole_Intrinsic::K(); the pair is kept iff it has more than 2.5 * 5 inliers.
// Robust_model_estimation_EAngular / _EUpright are GeometricFilter_ESphericalMatrix_AC_Angular<false / true>
// (E_ACRobust_Angular.hpp:52-160: eight-point / upright three-point essential matrix on bearing vectors, any camera type,
// spherical included): pairs whose views lack an intrinsic are skipped and not kept; the bearings are openMVG's own
// (*cam)(MatchesPairToMat(...)); all pairs go to omvg_geom_angular_acransac in one call (AC-RANSAC, then
// RelativePoseFromEssential), and a pair is kept iff its list has more than 2.5 * 8 (2.5 * 3) entries.  With
// b_guided_matching the reference's Geometry_guided_matching of this functor only logs "Not yet implemented" and the
// pair is inserted with the EMPTY list it leaves (GeometricFilter.hpp:103-116); the shim does the same, logging once.
//
// Guided matching (b_guided_matching, openMVG_main_GeometricFilter's -r; GeometricFilter.hpp:96-123): the kept pairs go
// through geometry_aware::GuidedMatching on the device in ONE omvg_match_guided_run call, and its result replaces the
// AC-RANSAC inliers (a possibly empty list is still inserted, as the reference inserts it).  The descriptors and the
// un-distorted positions (openMVG's own get_ud_pixel, once per image) of the views in kept pairs go into one match
// context.  Model: F; for E, F = K_J^-T E K_I^-1 as FundamentalFromEssential forms it; for H, the homography.  Threshold Square(errorMax),
// distance ratio Square(d_distance_ratio), or the descriptor-free variant for H with a negative ratio followed by
// IndMatch::getDeduplicated and IndMatchDecorator<float>::getDeduplicated (H_ACRobust.hpp:136-202).  Regions other than
// 128-byte unsigned char descriptors are not supported: the call logs and returns false.
// Header-only; compile inside an openMVG build and link libomvg_b200.so.
#ifndef OPENMVG_B200_GEOMETRIC_FILTER_B200_HPP
#define OPENMVG_B200_GEOMETRIC_FILTER_B200_HPP

#include "openMVG/cameras/Camera_Common.hpp"
#include "openMVG/cameras/Camera_Pinhole.hpp"
#include "openMVG/matching/indMatch.hpp"
#include "openMVG/matching/indMatchDecoratorXY.hpp"
#include "openMVG/matching_image_collection/Geometric_Filter_utils.hpp"
#include "openMVG/sfm/pipelines/sfm_regions_provider.hpp"
#include "openMVG/sfm/sfm_data.hpp"
#include "openMVG/system/logger.hpp"
#include "openMVG/system/progressinterface.hpp"

#include "omvg_b200.h"

#include <cmath>
#include <map>
#include <memory>
#include <typeinfo>
#include <vector>

namespace openMVG {
namespace matching_image_collection {

struct ImageCollectionGeometricFilter_B200
{
  ImageCollectionGeometricFilter_B200(const sfm::SfM_Data * sfm_data, const std::shared_ptr<sfm::Regions_Provider> & regions_provider, int device = 0)
    : sfm_data_(sfm_data), regions_provider_(regions_provider), device_(device) {}

  // F model, a-contrario (GeometricFilter_FMatrix_AC(dPrecision, iteration)); returns false on a device error
  bool Robust_model_estimation_F(const matching::PairWiseMatches & putative_matches, double dPrecision = 4.0, uint32_t iteration = 2048,
                                 system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false, double d_distance_ratio = 0.6)
  { return Robust_model_estimation(OMVG_GEOM_FUNDAMENTAL, putative_matches, dPrecision, iteration, my_progress_bar, b_guided_matching, d_distance_ratio); }
  // H model (GeometricFilter_HMatrix_AC(dPrecision, iteration), H_ACRobust.hpp:46-112): kept iff more than 2.5 * 4 inliers
  bool Robust_model_estimation_H(const matching::PairWiseMatches & putative_matches, double dPrecision = 4.0, uint32_t iteration = 2048,
                                 system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false, double d_distance_ratio = 0.6)
  { return Robust_model_estimation(OMVG_GEOM_HOMOGRAPHY, putative_matches, dPrecision, iteration, my_progress_bar, b_guided_matching, d_distance_ratio); }
  // E model (GeometricFilter_EMatrix_AC(dPrecision, iteration), E_ACRobust.hpp:55-150): kept iff more than 2.5 * 5 inliers
  bool Robust_model_estimation_E(const matching::PairWiseMatches & putative_matches, double dPrecision = 4.0, uint32_t iteration = 2048,
                                 system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false, double d_distance_ratio = 0.6)
  { return Robust_model_estimation(OMVG_GEOM_ESSENTIAL, putative_matches, dPrecision, iteration, my_progress_bar, b_guided_matching, d_distance_ratio); }

  // angular E models (GeometricFilter_ESphericalMatrix_AC_Angular<false | true>(dPrecision, iteration)): dPrecision in
  // degrees; kept iff more than 2.5 * 8 (eight-point) or 2.5 * 3 (upright) entries after the cheirality step
  bool Robust_model_estimation_EAngular(const matching::PairWiseMatches & putative_matches, double dPrecision = 4.0, uint32_t iteration = 2048,
                                        system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false, double d_distance_ratio = 0.6)
  { return Robust_model_estimation_Angular(false, putative_matches, dPrecision, iteration, my_progress_bar, b_guided_matching); }
  bool Robust_model_estimation_EUpright(const matching::PairWiseMatches & putative_matches, double dPrecision = 4.0, uint32_t iteration = 2048,
                                        system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false, double d_distance_ratio = 0.6)
  { return Robust_model_estimation_Angular(true, putative_matches, dPrecision, iteration, my_progress_bar, b_guided_matching); }

  bool Robust_model_estimation_Angular(bool upright, const matching::PairWiseMatches & putative_matches, double dPrecision, uint32_t iteration,
                                       system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false)
  {
    if (!my_progress_bar) my_progress_bar = &system::ProgressInterface::dummy();
    my_progress_bar->Restart(putative_matches.size(), "- Geometric filtering (B200) -");
    std::vector<uint64_t> offsets(1, 0);
    std::vector<double> bI, bJ;
    std::vector<const std::pair<const Pair, matching::IndMatches> *> order;
    size_t skipped = 0;
    for (const auto & it : putative_matches)
    {
      const cameras::IntrinsicBase * cam[2] = {nullptr, nullptr};    // E_ACRobust_Angular.hpp:78-99
      const IndexT ids[2] = {it.first.first, it.first.second};
      for (int k = 0; k < 2; ++k)
      {
        const IndexT id_intrinsic = sfm_data_->views.at(ids[k])->id_intrinsic;
        if (sfm_data_->GetIntrinsics().count(id_intrinsic)) cam[k] = sfm_data_->GetIntrinsics().at(id_intrinsic).get();
      }
      if (!cam[0] || !cam[1])
      {
        ++skipped;
        continue;
      }
      Mat2X a, b;
      MatchesPairToMat(it.first, it.second, sfm_data_, regions_provider_, a, b);
      const Mat3X ba = (*cam[0])(a), bb = (*cam[1])(b);               // E_ACRobust_Angular.hpp:105-107
      for (Mat3X::Index k = 0; k < ba.cols(); ++k)
        for (int c = 0; c < 3; ++c) { bI.push_back(ba(c, k)); bJ.push_back(bb(c, k)); }
      offsets.push_back(offsets.back() + static_cast<uint64_t>(ba.cols()));
      order.push_back(&it);
    }
    const size_t n_pairs = order.size();
    std::vector<uint32_t> inliers(bI.size() / 3 + 1);
    n_inliers_.assign(n_pairs + 1, 0); F_.assign(9 * n_pairs, 0.0); stats_.assign(2 * n_pairs, 0.0);
    _map_GeometricMatches.clear();
    const int rc = omvg_geom_angular_acransac(device_, upright ? OMVG_GEOM_ESSENTIAL_UPRIGHT : OMVG_GEOM_ESSENTIAL_ANGULAR, n_pairs, offsets.data(),
                                              bI.data(), bJ.data(), dPrecision, iteration, inliers.data(), n_inliers_.data(), F_.data(),
                                              stats_.data(), nullptr, nullptr);
    for (size_t p = 0; p < skipped; ++p) ++(*my_progress_bar);
    if (rc != OMVG_OK)
    {
      OPENMVG_LOG_ERROR << "omvg_b200: " << omvg_last_error();
      return false;
    }
    const double min_samples = upright ? 3.0 : 8.0;
    bool logged = false;
    for (size_t p = 0; p < n_pairs; ++p)
    {
      if (n_inliers_[p] > min_samples * 2.5)                       // E_ACRobust_Angular.hpp:146
      {
        matching::IndMatches geometric_inliers;
        if (b_guided_matching)
        {
          if (!logged) OPENMVG_LOG_ERROR << "Not yet implemented";  // the functor's Geometry_guided_matching
          logged = true;
        }
        else
        {
          geometric_inliers.reserve(n_inliers_[p]);
          for (uint32_t k = 0; k < n_inliers_[p]; ++k) geometric_inliers.push_back(order[p]->second[inliers[offsets[p] + k]]);
        }
        _map_GeometricMatches.insert({order[p]->first, std::move(geometric_inliers)});
      }
      ++(*my_progress_bar);
    }
    n_inliers_.resize(n_pairs);
    return true;
  }

  bool Robust_model_estimation(int32_t model, const matching::PairWiseMatches & putative_matches, double dPrecision, uint32_t iteration,
                               system::ProgressInterface * my_progress_bar = nullptr, bool b_guided_matching = false, double d_distance_ratio = 0.6)
  {
    if (!my_progress_bar) my_progress_bar = &system::ProgressInterface::dummy();
    my_progress_bar->Restart(putative_matches.size(), "- Geometric filtering (B200) -");
    std::vector<uint64_t> offsets(1, 0);
    std::vector<double> xI, xJ;
    std::vector<int32_t> size;
    std::vector<double> intr;                                   // E: f, ppx, ppy of view I then view J, per pair sent
    std::vector<const std::pair<const Pair, matching::IndMatches> *> order;
    const bool essential = model == OMVG_GEOM_ESSENTIAL;
    size_t skipped = 0;
    for (const auto & it : putative_matches)
    {
      if (essential)                                            // E_ACRobust.hpp:74-98
      {
        const cameras::IntrinsicBase * cam[2] = {nullptr, nullptr};
        const IndexT ids[2] = {it.first.first, it.first.second};
        for (int k = 0; k < 2; ++k)
        {
          const IndexT id_intrinsic = sfm_data_->views.at(ids[k])->id_intrinsic;
          if (sfm_data_->GetIntrinsics().count(id_intrinsic)) cam[k] = sfm_data_->GetIntrinsics().at(id_intrinsic).get();
        }
        if (!cam[0] || !cam[1] || !cameras::isPinhole(cam[0]->getType()) || !cameras::isPinhole(cam[1]->getType()))
        {
          ++skipped;
          continue;
        }
        for (int k = 0; k < 2; ++k)
        {
          const Mat3 & K = dynamic_cast<const cameras::Pinhole_Intrinsic *>(cam[k])->K();
          intr.insert(intr.end(), {K(0, 0), K(0, 2), K(1, 2)});
        }
      }
      Mat2X a, b;
      MatchesPairToMat(it.first, it.second, sfm_data_, regions_provider_, a, b);
      for (Mat2X::Index k = 0; k < a.cols(); ++k) { xI.push_back(a(0, k)); xI.push_back(a(1, k)); xJ.push_back(b(0, k)); xJ.push_back(b(1, k)); }
      offsets.push_back(offsets.back() + static_cast<uint64_t>(a.cols()));
      const sfm::View * vI = sfm_data_->GetViews().at(it.first.first).get(), * vJ = sfm_data_->GetViews().at(it.first.second).get();
      size.insert(size.end(), {static_cast<int32_t>(vI->ui_width), static_cast<int32_t>(vI->ui_height), static_cast<int32_t>(vJ->ui_width), static_cast<int32_t>(vJ->ui_height)});
      order.push_back(&it);
    }
    const size_t n_pairs = order.size();
    std::vector<uint32_t> inliers(xI.size() / 2 + 1), n_inliers(n_pairs + 1);
    F_.assign(9 * n_pairs, 0.0); stats_.assign(2 * n_pairs, 0.0);
    _map_GeometricMatches.clear();
    const double min_samples = model == OMVG_GEOM_FUNDAMENTAL ? 7.0 : essential ? 5.0 : 4.0;
    const int rc = essential
      ? omvg_geom_essential_acransac(device_, n_pairs, offsets.data(), xI.data(), xJ.data(), size.data(), intr.data(), dPrecision, iteration,
                                     inliers.data(), n_inliers.data(), F_.data(), stats_.data())
      : omvg_geom_acransac(device_, model, n_pairs, offsets.data(), xI.data(), xJ.data(), size.data(), dPrecision, iteration,
                           inliers.data(), n_inliers.data(), F_.data(), stats_.data());
    for (size_t p = 0; p < skipped; ++p) ++(*my_progress_bar);
    if (rc != OMVG_OK)
    {
      OPENMVG_LOG_ERROR << "omvg_b200: " << omvg_last_error();
      return false;
    }
    std::vector<size_t> kept;
    for (size_t p = 0; p < n_pairs; ++p)
    {
      if (n_inliers[p] > min_samples * 2.5)                      // F_ACRobust.hpp:85, H_ACRobust.hpp:97, E_ACRobust.hpp:135
      {
        if (b_guided_matching)
          kept.push_back(p);
        else
        {
          matching::IndMatches geometric_inliers;
          geometric_inliers.reserve(n_inliers[p]);
          for (uint32_t k = 0; k < n_inliers[p]; ++k) geometric_inliers.push_back(order[p]->second[inliers[offsets[p] + k]]);
          _map_GeometricMatches.insert({order[p]->first, std::move(geometric_inliers)});
        }
      }
      ++(*my_progress_bar);
    }
    if (b_guided_matching) return Guided_matching(model, order, intr, kept, d_distance_ratio);
    return true;
  }

  // geometry_aware::GuidedMatching of the kept pairs (the Geometry_guided_matching of F_ACRobust.hpp:109-151,
  // E_ACRobust.hpp:153-214, H_ACRobust.hpp:136-202) in one device call; the results replace the pairs' inliers
  bool Guided_matching(int32_t model, const std::vector<const std::pair<const Pair, matching::IndMatches> *> & order,
                       const std::vector<double> & intr, const std::vector<size_t> & kept, double d_distance_ratio)
  {
    std::map<IndexT, uint32_t> dense;                            // view id -> image of the match context
    std::vector<std::shared_ptr<features::Regions>> regions;
    std::vector<const cameras::IntrinsicBase *> cams;
    std::vector<uint32_t> pi, pj;
    std::vector<double> models, thresholds;
    std::vector<size_t> sent;
    for (const size_t p : kept)
    {
      const double thr = Square(stats_[2 * p]);
      if (!std::isfinite(thr)) { _map_GeometricMatches.insert({order[p]->first, matching::IndMatches()}); continue; }   // precision = infinity: no guided step
      const IndexT ids[2] = {order[p]->first.first, order[p]->first.second};
      uint32_t img[2];
      for (int k = 0; k < 2; ++k)
      {
        auto it = dense.find(ids[k]);
        if (it == dense.end())
        {
          std::shared_ptr<features::Regions> r = regions_provider_->get(ids[k]);
          if (!r || !r->IsScalar() || r->Type_id() != typeid(unsigned char).name() || r->DescriptorLength() != OMVG_DESC_LEN)
          {
            OPENMVG_LOG_ERROR << "omvg_b200: guided matching needs 128-byte unsigned char descriptors (view " << ids[k] << ")";
            return false;
          }
          const sfm::View * v = sfm_data_->GetViews().at(ids[k]).get();
          cams.push_back(sfm_data_->GetIntrinsics().count(v->id_intrinsic) ? sfm_data_->GetIntrinsics().at(v->id_intrinsic).get() : nullptr);
          regions.push_back(r);
          it = dense.insert({ids[k], static_cast<uint32_t>(regions.size() - 1)}).first;
        }
        img[k] = it->second;
      }
      Mat3 M;
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M(r, c) = F_[9 * p + 3 * r + c];
      if (model == OMVG_GEOM_ESSENTIAL)                           // E_ACRobust.hpp:199-200
      {
        const double * k6 = &intr[6 * p];
        Mat3 KI, KJ;
        KI << k6[0], 0, k6[1], 0, k6[0], k6[2], 0, 0, 1;          // Pinhole_Intrinsic::K()
        KJ << k6[3], 0, k6[4], 0, k6[3], k6[5], 0, 0, 1;
        // FundamentalFromEssential(E, K_I, K_J, &F) (multiview/essential.cpp:48-53), the same expression written out
        // so that this header needs no symbol of openMVG_multiview
        const Mat3 F = KJ.inverse().transpose() * M * KI.inverse();
        M = F;
      }
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) models.push_back(M(r, c));
      thresholds.push_back(thr);
      pi.push_back(img[0]); pj.push_back(img[1]); sent.push_back(p);
    }
    const bool geometry_only = model == OMVG_GEOM_HOMOGRAPHY && d_distance_ratio < 0;
    const double ratio = geometry_only ? -1.0 : Square(d_distance_ratio);
    std::vector<uint32_t> counts(regions.size());
    for (size_t k = 0; k < regions.size(); ++k) counts[k] = static_cast<uint32_t>(regions[k]->RegionCount());
    omvg_match_ctx * ctx = nullptr;
    const uint64_t * off = nullptr; const uint32_t * ij = nullptr; uint64_t n_matches = 0;
    int rc = omvg_match_create(&ctx, device_);
    if (rc == OMVG_OK) rc = omvg_match_set_images(ctx, static_cast<uint32_t>(counts.size()), counts.data());
    for (size_t k = 0; k < regions.size() && rc == OMVG_OK; ++k)
    {
      std::vector<double> xy(2 * counts[k]);
      for (uint32_t f = 0; f < counts[k]; ++f)                   // guided_matching.hpp:196-201
      {
        const Vec2 x = cams[k] ? cams[k]->get_ud_pixel(regions[k]->GetRegionPosition(f)) : regions[k]->GetRegionPosition(f);
        xy[2 * f] = x(0); xy[2 * f + 1] = x(1);
      }
      rc = omvg_match_upload_host(ctx, static_cast<uint32_t>(k), static_cast<const uint8_t *>(regions[k]->DescriptorRawData()));
      if (rc == OMVG_OK) rc = omvg_match_upload_positions(ctx, static_cast<uint32_t>(k), xy.data());
    }
    if (rc == OMVG_OK) rc = omvg_match_prepare(ctx);
    if (rc == OMVG_OK) rc = omvg_match_guided_run(ctx, model == OMVG_GEOM_HOMOGRAPHY ? OMVG_GUIDED_TRANSFER : OMVG_GUIDED_EPIPOLAR,
                                                  pi.data(), pj.data(), pi.size(), models.data(), thresholds.data(), ratio);
    if (rc == OMVG_OK) rc = omvg_match_fetch(ctx, &off, &ij, &n_matches);
    if (rc != OMVG_OK)
    {
      OPENMVG_LOG_ERROR << "omvg_b200: " << omvg_last_error();
      omvg_match_destroy(ctx);
      return false;
    }
    for (size_t q = 0; q < sent.size(); ++q)
    {
      matching::IndMatches m;
      for (uint64_t k = off[q]; k < off[q + 1]; ++k) m.emplace_back(ij[2 * k], ij[2 * k + 1]);
      matching::IndMatch::getDeduplicated(m);
      if (geometry_only)                                          // H_ACRobust.hpp:176-182
      {
        matching::IndMatchDecorator<float> deduplicator(m, regions[pi[q]]->GetRegionsPositions(), regions[pj[q]]->GetRegionsPositions());
        deduplicator.getDeduplicated(m);
      }
      _map_GeometricMatches.insert({order[sent[q]]->first, std::move(m)});
    }
    omvg_match_destroy(ctx);
    return true;
  }

  const matching::PairWiseMatches & Get_geometric_matches() const { return _map_GeometricMatches; }

  const sfm::SfM_Data * sfm_data_;
  const std::shared_ptr<sfm::Regions_Provider> regions_provider_;   // (a copy: the reference keeps a reference, which dangles when bound to a converted temporary)
  int device_;
  matching::PairWiseMatches _map_GeometricMatches;
  std::vector<double> F_, stats_;                               // per pair sent (map order): un-normalised F (H, E), {errorMax, minNFA}
  std::vector<uint32_t> n_inliers_;                             // angular models, per pair sent: the list length after the cheirality step
};

}  // namespace matching_image_collection
}  // namespace openMVG

#endif  // OPENMVG_B200_GEOMETRIC_FILTER_B200_HPP
