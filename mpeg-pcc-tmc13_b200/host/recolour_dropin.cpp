// recolour_dropin.cpp — host-side mirror of the reference interface for
// recolouring: a translation unit that DEFINES the reference's own entry point
//
//   pcc::recolour                       (tmc3/pointset_processing.h:194,
//                                        tmc3/pointset_processing.cpp:925-958)
//
// with its exact C++ signature and forwards it to pccb200_recolour_exact, the
// library's reference-exact recolouring (nanoflann's trees and search, the
// std::sort list order).  The caller, the encoder's recolouring of every
// attribute set when geometry coding adds or removes points
// (tmc3/encoder.cpp:1029-1037), is unchanged, and the bitstream stays
// byte-identical (tests/test_recolour_exact.py::test_whole_codec_recolour).
//
// The side effects are the reference's: the target gains colours
// (addColors) or reflectances (addReflectances), a missing source attribute or
// an empty cloud returns -1, and any other attribute label is left alone.  The
// scale arrives as a float and becomes a double as the reference's call of
// recolourColour / recolourReflectance converts it.
//
// It is linked INSTEAD of the reference's definition: oracle/recolour_codec.mk
// renames that one symbol in pointset_processing.o (objcopy --redefine-sym) to
// pccb200_reference_recolour, which this unit keeps for the parameters the
// library does not take (more than 16 neighbours or more neighbours than
// points, a search range above 8, bit depths outside 1..16, other attribute
// widths, coordinates of |x| >= 2^30).  With PCCB200_DROPIN_STRICT=1 in the
// environment those throw instead, so that a run proves the library did the
// work.  A maintainer would instead rename the function in
// pointset_processing.cpp; see INTEGRATION.md.
#include <cstdlib>
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "pointset_processing.h"

#include "pcc_attr_b200.h"

namespace pcc {

// the reference's own recolour under its link-time name
extern "C" int pccb200_reference_recolour(
  const AttributeDescription& desc, const RecolourParams& cfg, const PCCPointSet3& source,
  float sourceToTargetScaleFactor, point_t tgtToSrcOffset, PCCPointSet3* target);

namespace {

bool
strict()
{
  const char* s = std::getenv("PCCB200_DROPIN_STRICT");
  return s && s[0] == '1';
}

bool
coords_in_range(const PCCPointSet3& c)
{
  for (size_t i = 0; i < c.getPointCount(); i++)
    for (int k = 0; k < 3; k++)
      if (c[i][k] <= -(1 << 30) || c[i][k] >= (1 << 30))
        return false;
  return true;
}

}  // namespace

int
recolour(
  const AttributeDescription& desc,
  const RecolourParams& cfg,
  const PCCPointSet3& source,
  float sourceToTargetScaleFactor,
  point_t tgtToSrcOffset,
  PCCPointSet3* target)
{
  const bool colour = desc.attributeLabel == KnownAttributeLabel::kColour;
  const bool refl = desc.attributeLabel == KnownAttributeLabel::kReflectance;
  if (!colour && !refl)
    return 0;
  const int A = colour ? 3 : 1;
  const int64_t ns = int64_t(source.getPointCount());
  const int64_t nt = int64_t(target->getPointCount());
  const double scale = sourceToTargetScaleFactor;
  bool covered = ns > 0 && nt > 0 && ns < (int64_t(1) << 31) && nt < (int64_t(1) << 31)
    && (colour ? source.hasColors() : source.hasReflectances())
    && int(desc.attr_num_dimensions_minus1) + 1 == A && desc.bitdepth >= 1 && desc.bitdepth <= 16
    && cfg.numNeighboursFwd >= 1 && cfg.numNeighboursFwd <= 16 && cfg.numNeighboursFwd <= ns
    && cfg.numNeighboursBwd >= 1 && cfg.numNeighboursBwd <= 16 && cfg.numNeighboursBwd <= nt
    && cfg.searchRange >= 0 && cfg.searchRange <= 8 && scale > 0.0;
  for (int k = 0; k < 3 && covered; k++)
    covered = tgtToSrcOffset[k] > -(1 << 30) && tgtToSrcOffset[k] < (1 << 30);
  covered = covered && coords_in_range(source) && coords_in_range(*target);
  if (!covered) {
    if (strict())
      throw std::runtime_error("recolour drop-in: parameters outside the library's range");
    return pccb200_reference_recolour(
      desc, cfg, source, sourceToTargetScaleFactor, tgtToSrcOffset, target);
  }

  std::vector<int32_t> sxyz(3 * ns), sattr(A * ns), txyz(3 * nt), out(A * nt);
  for (int64_t i = 0; i < ns; i++) {
    for (int k = 0; k < 3; k++)
      sxyz[3 * i + k] = source[i][k];
    if (colour) {
      const Vec3<attr_t> c = source.getColor(i);
      for (int k = 0; k < 3; k++)
        sattr[3 * i + k] = c[k];
    } else {
      sattr[i] = source.getReflectance(i);
    }
  }
  for (int64_t i = 0; i < nt; i++)
    for (int k = 0; k < 3; k++)
      txyz[3 * i + k] = (*target)[i][k];

  pccb200_recolour_params p;
  p.dist_offset_fwd = cfg.distOffsetFwd;
  p.dist_offset_bwd = cfg.distOffsetBwd;
  p.max_geometry_dist2_fwd = cfg.maxGeometryDist2Fwd;
  p.max_geometry_dist2_bwd = cfg.maxGeometryDist2Bwd;
  p.max_attribute_dist2_fwd = cfg.maxAttributeDist2Fwd;
  p.max_attribute_dist2_bwd = cfg.maxAttributeDist2Bwd;
  p.search_range = cfg.searchRange;
  p.num_neighbours_fwd = cfg.numNeighboursFwd;
  p.num_neighbours_bwd = cfg.numNeighboursBwd;
  p.use_dist_weighted_avg_fwd = cfg.useDistWeightedAvgFwd;
  p.use_dist_weighted_avg_bwd = cfg.useDistWeightedAvgBwd;
  p.skip_avg_if_identical_source_point_present_fwd = cfg.skipAvgIfIdenticalSourcePointPresentFwd;
  p.skip_avg_if_identical_source_point_present_bwd = cfg.skipAvgIfIdenticalSourcePointPresentBwd;
  p.reserved = 0;
  const int32_t off[3] = {tgtToSrcOffset[0], tgtToSrcOffset[1], tgtToSrcOffset[2]};
  const int rc = pccb200_recolour_exact(
    &p, sxyz.data(), sattr.data(), A, int32_t(ns), scale, off, txyz.data(), int32_t(nt),
    desc.bitdepth, out.data());
  if (rc != PCCB200_OK) {
    if (strict())
      throw std::runtime_error(
        std::string("recolour drop-in: pccb200_recolour_exact failed: ") + pccb200_last_error());
    return pccb200_reference_recolour(
      desc, cfg, source, sourceToTargetScaleFactor, tgtToSrcOffset, target);
  }

  if (colour) {
    target->addColors();
    for (int64_t i = 0; i < nt; i++)
      target->setColor(
        i, Vec3<attr_t>(attr_t(out[3 * i]), attr_t(out[3 * i + 1]), attr_t(out[3 * i + 2])));
  } else {
    target->addReflectances();
    for (int64_t i = 0; i < nt; i++)
      target->setReflectance(i, attr_t(out[i]));
  }
  return 0;
}

}  // namespace pcc
