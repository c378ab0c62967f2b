// ref_shim_scalable_enc.cpp — TEST INFRASTRUCTURE ONLY (oracle).
//
// Scalable lifting (aps.scalable_lifting_enabled_flag) through the reference's
// own code, as ref_shim_liftenc.cpp reaches the lifting encoder: this TU
// #includes tmc3/AttributeEncoder.cpp from where it lies, with `protected` /
// `private` opened.
//   tmc13ref_scalable_lod_build    AttributeLods::generate
//                                  (tmc3/AttributeCommon.cpp:45-72) with the
//                                  flag and a given minGeomNodeSizeLog2
//   tmc13ref_scalable_lift_encode  encode{Colors,Reflectances}Lift
//                                  (tmc3/AttributeEncoder.cpp:1379-1648)
//   tmc13ref_scalable_payload      a quantised value stream through the
//                                  reference's PCCResidualsEncoder, for the
//                                  decoder of ref_shim_scalable_dec.cpp
// Built by oracle/scalable.mk into _ref/libtmc13_scalable.so.
// standard headers first: opening `private` must not reach libstdc++
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <list>
#include <map>
#include <memory>
#include <numeric>
#include <queue>
#include <set>
#include <sstream>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>
#define protected public
#define private public
#include "AttributeEncoder.cpp"
#undef protected
#undef private

#include "pcc_attr_b200.h"

using namespace pcc;

// the APS of a scalable lifting slice, as tmc3/TMC3.cpp:2113-2125 requires it
// (lod_decimation_type 0; num_detail_levels and dist2 are not read)
void
tmc13ref_scalable_aps(const pccb200_lod_params* lp, int maxNeighRange, AttributeParameterSet& aps)
{
  aps.attr_encoding = AttributeEncoding::kLiftingTransform;
  aps.lod_decimation_type = LodDecimationMethod(lp->lod_decimation_type);
  aps.canonical_point_order_flag = false;
  aps.max_points_per_sort_log2_plus1 = 0;
  aps.num_pred_nearest_neighbours_minus1 = lp->num_pred_nearest_neighbours - 1;
  aps.num_detail_levels_minus1 = lp->num_detail_levels - 1;
  aps.dist2 = lp->dist2;
  aps.inter_lod_search_range = lp->inter_lod_search_range;
  aps.intra_lod_search_range = lp->intra_lod_search_range;
  aps.intra_lod_prediction_skip_layers = lp->intra_lod_prediction_skip_layers;
  aps.predictionWithDistributionEnabled = lp->prediction_with_distribution != 0;
  aps.lodNeighBias = {lp->lod_neigh_bias[0], lp->lod_neigh_bias[1], lp->lod_neigh_bias[2]};
  aps.pred_weight_blending_enabled_flag = lp->pred_weight_blending != 0;
  aps.scalable_lifting_enabled_flag = true;
  aps.max_neigh_range_minus1 = maxNeighRange - 1;
  aps.lodSamplingPeriod.assign(
    lp->lod_sampling_period, lp->lod_sampling_period + PCCB200_MAX_LODS);
}

static AttributeInterPredParams
intra()
{
  AttributeInterPredParams ip;
  ip.frameDistance = 1;
  ip.enableAttrInterPred = false;
  ip.attrInterIntraSliceRDO = false;
  return ip;
}

static void
lods_out(
  const AttributeLods& lods, int n, pccb200_predictor* predsOut, uint32_t* indexesOut,
  uint32_t* numPointsInLodOut, int32_t* lodCountOut)
{
  for (int i = 0; i < n; i++) {
    const auto& p = lods.predictors[i];
    predsOut[i].neighbor_count = p.neighborCount;
    for (int j = 0; j < 3; j++) {
      predsOut[i].predictor_index[j] = j < int(p.neighborCount) ? p.neighbors[j].predictorIndex : 0;
      predsOut[i].weight[j] = j < int(p.neighborCount) ? uint32_t(p.neighbors[j].weight) : 0;
    }
    indexesOut[i] = lods.indexes[i];
  }
  *lodCountOut = int(lods.numPointsInLod.size());
  for (size_t i = 0; i < lods.numPointsInLod.size() && i < PCCB200_MAX_LODS; i++)
    numPointsInLodOut[i] = lods.numPointsInLod[i];
}

// geomNumPoints: geom_num_points_minus1 + 1 (>= n; the points a partial decode
// skipped make up the difference)
extern "C" void
tmc13ref_scalable_lod_build(
  const pccb200_lod_params* lp, int maxNeighRange, int minGeomNodeSizeLog2, int geomNumPoints,
  const int32_t* xyz, int n, pccb200_predictor* predsOut, uint32_t* indexesOut,
  uint32_t* numPointsInLodOut, int32_t* lodCountOut)
{
  AttributeParameterSet aps{};
  tmc13ref_scalable_aps(lp, maxNeighRange, aps);
  AttributeBrickHeader abh{};
  PCCPointSet3 cloud;
  cloud.resize(n);
  for (int i = 0; i < n; i++)
    cloud[i] = point_t{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  AttributeLods lods;
  lods.generate(aps, abh, geomNumPoints - 1, minGeomNodeSizeLog2, cloud, intra());
  lods_out(lods, n, predsOut, indexesOut, numPointsInLodOut, lodCountOut);
}

extern "C" int tmc13ref_scalable_decode_values(
  const uint8_t* buf, int len, int n, int numAttrs, int32_t* valuesOut);

static QpSet
qpset_of(const pccb200_qpset* qs)
{
  QpSet qpSet;
  for (int i = 0; i < qs->num_layers; i++)
    qpSet.layers.push_back(Qps{qs->layers[i][0], qs->layers[i][1]});
  qpSet.maxQp = qs->max_qp;
  qpSet.fixedPointQpOffset = qs->fixed_point_qp_offset;
  return qpSet;
}

// the encoder's generate (geom_num_points_minus1 = n - 1, minGeomNodeSizeLog2
// = 0) and lifting body.  lcpOut: 21 entries (colour only).
extern "C" void
tmc13ref_scalable_lift_encode(
  const pccb200_lod_params* lp, int maxNeighRange, const pccb200_qpset* qs, int lcpEnabled,
  const int32_t* xyz, const int32_t* attrs, int n, int numAttrs, int bitdepth,
  int32_t* valuesOut, int32_t* reconOut, int8_t* lcpOut)
{
  AttributeParameterSet aps{};
  tmc13ref_scalable_aps(lp, maxNeighRange, aps);
  aps.last_component_prediction_enabled_flag = lcpEnabled != 0;
  AttributeBrickHeader abh{};
  AttributeDescription desc{};
  desc.bitdepth = bitdepth;
  desc.attr_num_dimensions_minus1 = numAttrs - 1;
  SequenceParameterSet sps{};
  QpSet qpSet = qpset_of(qs);

  PCCPointSet3 cloud;
  cloud.addRemoveAttributes(numAttrs == 3, numAttrs == 1);
  cloud.resize(n);
  for (int i = 0; i < n; i++) {
    cloud[i] = point_t{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
    if (numAttrs == 3)
      cloud.setColor(i, Vec3<attr_t>(attrs[3 * i], attrs[3 * i + 1], attrs[3 * i + 2]));
    else
      cloud.setReflectance(i, attr_t(attrs[i]));
  }
  AttributeInterPredParams ip = intra();
  AttributeEncoder enc;
  enc._abh = &abh;
  enc._lods.generate(aps, abh, n - 1, 0, cloud, ip);
  AttributeContexts ctxtMem;
  ctxtMem.reset();
  PCCResidualsEncoder encoder(aps, abh, ctxtMem);
  encoder.start(sps, n);
  if (numAttrs == 3)
    enc.encodeColorsLift(desc, aps, qpSet, cloud, encoder);
  else
    enc.encodeReflectancesLift(desc, aps, qpSet, cloud, encoder, ip);
  int len = encoder.stop();
  tmc13ref_scalable_decode_values(
    reinterpret_cast<const uint8_t*>(encoder.arithmeticEncoder.buffer()), len, n, numAttrs,
    valuesOut);
  for (int i = 0; i < n; i++) {
    if (numAttrs == 3) {
      auto c = cloud.getColor(i);
      for (int k = 0; k < 3; k++)
        reconOut[3 * i + k] = c[k];
    } else {
      reconOut[i] = cloud.getReflectance(i);
    }
  }
  const int levels = aps.maxNumDetailLevels();
  if (lcpOut && numAttrs == 3)
    for (int l = 0; l < levels; l++)
      lcpOut[l] = l < int(abh.attrLcpCoeffs.size()) ? abh.attrLcpCoeffs[l] : 0;
}

// values (n x numAttrs, coding order) as the lifting encoder writes them
// (tmc3/AttributeEncoder.cpp:1461-1470).  Returns the payload length, or
// minus the length needed when cap is too small.
extern "C" int
tmc13ref_scalable_payload(const int32_t* values, int n, int numAttrs, uint8_t* buf, int cap)
{
  AttributeParameterSet aps{};
  aps.attr_encoding = AttributeEncoding::kLiftingTransform;
  AttributeBrickHeader abh{};
  SequenceParameterSet sps{};
  AttributeContexts ctxtMem;
  ctxtMem.reset();
  PCCResidualsEncoder encoder(aps, abh, ctxtMem);
  encoder.start(sps, n);
  int zeroRun = 0;
  for (int i = 0; i < n; i++) {
    const int32_t* v = &values[size_t(i) * numAttrs];
    bool zero = true;
    for (int k = 0; k < numAttrs; k++)
      zero = zero && !v[k];
    if (zero) {
      ++zeroRun;
      continue;
    }
    encoder.encodeRunLength(zeroRun);
    if (numAttrs == 3)
      encoder.encode(v[0], v[1], v[2]);
    else
      encoder.encode(v[0]);
    zeroRun = 0;
  }
  if (zeroRun)
    encoder.encodeRunLength(zeroRun);
  int len = encoder.stop();
  if (len > cap)
    return -len;
  memcpy(buf, encoder.arithmeticEncoder.buffer(), len);
  return len;
}
