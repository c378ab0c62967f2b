// ref_shim_preddec.cpp — TEST INFRASTRUCTURE ONLY (oracle).
//
// Runs the reference's own predicting-transform DECODER bodies
//   AttributeDecoder::decodeReflectancesPred  tmc3/AttributeDecoder.cpp:328-391
//   AttributeDecoder::decodeColorsPred        tmc3/AttributeDecoder.cpp:446-523
// on a payload of ref_shim_predenc.cpp, with the levels of detail the
// reference generates, and walks the same payload as those bodies do to return
// the values their entropy decoding yields (coding order, the prediction mode
// still in the low bits).  #includes the reference's AttributeDecoder.cpp from
// where it lies, as ref_shim_liftdec.cpp does.
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
#include "AttributeDecoder.cpp"
#undef protected
#undef private

#include "pcc_attr_b200.h"

using namespace pcc;

void
tmc13ref_pred_fill_aps(const pccb200_lod_params* lp, const pccb200_pred_params* pp,
                       const int32_t qnw[3], AttributeParameterSet& aps)
{
  aps.attr_encoding = AttributeEncoding::kPredictingTransform;
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
  aps.scalable_lifting_enabled_flag = false;
  aps.lodSamplingPeriod.assign(
    lp->lod_sampling_period, lp->lod_sampling_period + PCCB200_MAX_LODS);
  aps.max_num_direct_predictors = pp->max_num_direct_predictors;
  aps.direct_avg_predictor_disabled_flag = pp->direct_avg_predictor_disabled != 0;
  aps.adaptive_prediction_threshold = pp->adaptive_prediction_threshold;
  aps.inter_component_prediction_enabled_flag = pp->icp_enabled != 0;
  aps.last_component_prediction_enabled_flag = false;
  aps.quant_neigh_weight = Vec3<uint32_t>(qnw[0], qnw[1], qnw[2]);
}

extern "C" int
tmc13ref_pred_decode(
  const pccb200_lod_params* lp, const pccb200_qpset* qs, const pccb200_pred_params* pp,
  const int32_t* qnw, const int32_t* xyz, int n, int numAttrs, int bitdepth,
  const uint8_t* buf, int len,
  const int8_t* icp,       // PCCB200_MAX_LODS x 3, as the encoder wrote them
  int32_t* valuesOut,      // n x numAttrs, coding order
  int32_t* out)            // n x numAttrs, point order
{
  AttributeParameterSet aps{};
  tmc13ref_pred_fill_aps(lp, pp, qnw, aps);
  AttributeBrickHeader abh{};
  AttributeDescription desc{};
  desc.bitdepth = bitdepth;
  desc.attr_num_dimensions_minus1 = numAttrs - 1;
  SequenceParameterSet sps{};
  QpSet qpSet;
  for (int i = 0; i < qs->num_layers; i++)
    qpSet.layers.push_back(Qps{qs->layers[i][0], qs->layers[i][1]});
  qpSet.maxQp = qs->max_qp;
  qpSet.fixedPointQpOffset = qs->fixed_point_qp_offset;
  if (abh.icpPresent(desc, aps))
    for (int l = 0; l < PCCB200_MAX_LODS; l++)
      abh.icpCoeffs.push_back(Vec3<int8_t>(icp[3 * l], icp[3 * l + 1], icp[3 * l + 2]));

  PCCPointSet3 cloud;
  cloud.addRemoveAttributes(numAttrs == 3, numAttrs == 1);
  cloud.resize(n);
  for (int i = 0; i < n; i++)
    cloud[i] = point_t{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  AttributeInterPredParams ip;
  ip.frameDistance = 1;
  ip.enableAttrInterPred = false;
  ip.attrInterIntraSliceRDO = false;

  AttributeContexts ctxtMem;
  {
    // the values, walked as the bodies walk the payload
    ctxtMem.reset();
    PCCResidualsDecoder decoder(abh, ctxtMem);
    decoder.start(sps, reinterpret_cast<const char*>(buf), len);
    int zeroRunRem = 0;
    for (int i = 0; i < n; i++) {
      if (--zeroRunRem < 0)
        zeroRunRem = decoder.decodeRunLength();
      int32_t values[3] = {};
      if (!zeroRunRem) {
        if (numAttrs == 3)
          decoder.decode(values);
        else
          values[0] = decoder.decode();
      }
      for (int k = 0; k < numAttrs; k++)
        valuesOut[i * numAttrs + k] = values[k];
    }
    decoder.stop();
  }

  AttributeDecoder dec;
  dec._lods.generate(aps, abh, n - 1, 0, cloud, ip);
  ctxtMem.reset();
  PCCResidualsDecoder decoder(abh, ctxtMem);
  decoder.start(sps, reinterpret_cast<const char*>(buf), len);
  if (numAttrs == 3)
    dec.decodeColorsPred(desc, aps, abh, qpSet, decoder, cloud);
  else
    dec.decodeReflectancesPred(desc, aps, abh, qpSet, decoder, cloud, ip);
  decoder.stop();
  for (int i = 0; i < n; i++) {
    if (numAttrs == 3) {
      auto c = cloud.getColor(i);
      for (int k = 0; k < 3; k++)
        out[3 * i + k] = c[k];
    } else {
      out[i] = cloud.getReflectance(i);
    }
  }
  return 0;
}
