// lod_dropin.cpp — host-side mirror of the reference interface for the
// level-of-detail build of the predicting / lifting transforms: a translation
// unit that DEFINES the reference's own entry point
//
//   pcc::AttributeLods::generate        (tmc3/AttributeCommon.h:72-79,
//                                        tmc3/AttributeCommon.cpp:45-72)
//
// with its exact C++ signature and forwards it to the C ABI of
// libpcc_attr_b200.so (pccb200_lod_build / _scalable: Morton sort, subsampling, the
// nearest-neighbour search, predictor weights incl. blending).  The callers
// AttributeEncoder::encode (tmc3/AttributeEncoder.cpp:456-460) and
// AttributeDecoder::decode (tmc3/AttributeDecoder.cpp:229-233) are unchanged:
// they go on to run their coding loops on the predictors filled in here, and
// the bitstream stays byte-identical (tests/test_gpu_parity.py::
// test_whole_codec_bitstream_lifting).
//
// It is linked INSTEAD of the reference's definition: oracle/Makefile renames
// that one symbol in AttributeCommon.o (objcopy --redefine-sym) to
// pccb200_reference_lods_generate, which this unit keeps for the parameter
// combinations the library does not cover (canonical point order, inter-frame
// references).  Scalable lifting, partial decodes included, goes to
// pccb200_lod_build_scalable.  A maintainer would instead rename the
// function in AttributeCommon.cpp; see INTEGRATION.md.
#include <stdexcept>
#include <string>
#include <vector>

#include "AttributeCommon.h"

#include "pcc_attr_b200.h"

namespace pcc {

// the reference's own AttributeLods::generate under its link-time name
// (Itanium C++ ABI: a member function takes `this` as its first argument)
extern "C" void pccb200_reference_lods_generate(
  AttributeLods* self, const AttributeParameterSet& aps, const AttributeBrickHeader& abh,
  int geom_num_points_minus1, int minGeomNodeSizeLog2, const PCCPointSet3& cloud,
  const AttributeInterPredParams& attrInterPredParams);

void
AttributeLods::generate(
  const AttributeParameterSet& aps,
  const AttributeBrickHeader& abh,
  int geom_num_points_minus1,
  int minGeomNodeSizeLog2,
  const PCCPointSet3& cloud,
  const AttributeInterPredParams& attrInterPredParams)
{
  const int n = int(cloud.getPointCount());
  const bool scalable = aps.scalable_lifting_enabled_flag;
  // scalable lifting, including a partial decode (minGeomNodeSizeLog2 > 0)
  const bool levelsCovered = scalable
    ? int(aps.lod_decimation_type) == 0 && minGeomNodeSizeLog2 >= 0 && minGeomNodeSizeLog2 < 21
      && int64_t(geom_num_points_minus1) + 1 >= n
    : minGeomNodeSizeLog2 == 0 && aps.num_detail_levels_minus1 + 1 <= PCCB200_MAX_LODS;
  const bool covered = levelsCovered
    && !aps.canonical_point_order_flag && aps.max_points_per_sort_log2_plus1 == 0
    && !attrInterPredParams.enableAttrInterPred && n > 0
    && aps.num_pred_nearest_neighbours_minus1 < 3;
  if (!covered) {
    pccb200_reference_lods_generate(
      this, aps, abh, geom_num_points_minus1, minGeomNodeSizeLog2, cloud, attrInterPredParams);
    return;
  }

  _aps = aps;
  _abh = abh;

  pccb200_lod_params lp = {};
  lp.num_detail_levels = aps.num_detail_levels_minus1 + 1;
  lp.lod_decimation_type = int(aps.lod_decimation_type);
  for (int i = 0; i < PCCB200_MAX_LODS; i++)
    lp.lod_sampling_period[i] =
      i < int(aps.lodSamplingPeriod.size()) ? aps.lodSamplingPeriod[i] : 0;
  lp.dist2 = aps.dist2 + abh.attr_dist2_delta;
  lp.num_pred_nearest_neighbours = aps.num_pred_nearest_neighbours_minus1 + 1;
  lp.inter_lod_search_range = aps.inter_lod_search_range;
  lp.intra_lod_search_range = aps.intra_lod_search_range;
  lp.intra_lod_prediction_skip_layers = aps.intra_lod_prediction_skip_layers;
  lp.prediction_with_distribution = aps.predictionWithDistributionEnabled;
  for (int k = 0; k < 3; k++)
    lp.lod_neigh_bias[k] = aps.lodNeighBias[k];
  lp.pred_weight_blending = aps.attr_encoding == AttributeEncoding::kPredictingTransform
    && aps.pred_weight_blending_enabled_flag;

  std::vector<int32_t> xyz(size_t(n) * 3);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++)
      xyz[size_t(i) * 3 + k] = cloud[i][k];

  std::vector<pccb200_predictor> flat(n);
  indexes.resize(n);
  uint32_t npl[PCCB200_MAX_LODS] = {};
  int32_t lodCount = 0;
  pccb200_lod_scalable scal = {};
  scal.max_neigh_range = aps.max_neigh_range_minus1 + 1;
  scal.min_geom_node_size_log2 = minGeomNodeSizeLog2;
  scal.geom_num_points = int64_t(geom_num_points_minus1) + 1;
  int rc = scalable
    ? pccb200_lod_build_scalable(&lp, &scal, xyz.data(), n, flat.data(), indexes.data(), npl,
                                 &lodCount)
    : pccb200_lod_build(&lp, xyz.data(), n, flat.data(), indexes.data(), npl, &lodCount);
  if (rc != PCCB200_OK)
    throw std::runtime_error(
      std::string("pcc_attr_b200: LoD build failed: ") + pccb200_last_error());

  numPointsInLod.assign(npl, npl + lodCount);
  indexesRef.clear();
  numPointsInLodRef.clear();
  predictors.clear();
  predictors.resize(n);  // value-initialised: predMode 0
  for (int i = 0; i < n; i++) {
    PCCPredictor& p = predictors[i];
    p.init();
    p.neighborCount = flat[i].neighbor_count;
    for (uint32_t j = 0; j < p.neighborCount; j++) {
      PCCNeighborInfo& nb = p.neighbors[j];
      nb.predictorIndex = flat[i].predictor_index[j];
      nb.weight = flat[i].weight[j];
      nb.pointIndex = indexes[nb.predictorIndex];
      nb.interFrameRef = false;
    }
  }
}

}  // namespace pcc
