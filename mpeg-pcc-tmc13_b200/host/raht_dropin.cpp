// raht_dropin.cpp — host-side mirror of the reference interface for the RAHT
// path: a translation unit that DEFINES the reference's own entry points
//
//   pcc::regionAdaptiveHierarchicalTransform         (tmc3/RAHT.h:47-57)
//   pcc::regionAdaptiveHierarchicalInverseTransform  (tmc3/RAHT.h:59-69)
//
// with their exact C++ signatures and forwards them to the C ABI of
// libpcc_attr_b200.so.  It is compiled inside the TMC13 tree INSTEAD of
// tmc3/RAHT.cpp (it includes the reference's headers, it does not copy them);
// AttributeEncoder.cpp:1273,1341 and AttributeDecoder.cpp:595,658 then call the
// CUDA path unchanged.  See INTEGRATION.md.
//
// Error behaviour mirrors the reference: the functions return void; failures
// (no device, CUDA error, inter-frame prediction requested) throw
// std::runtime_error like tmc3/encoder.cpp:1025 does for level limits.
#include <stdexcept>
#include <string>
#include <vector>

#include "RAHT.h"

#include "pcc_attr_b200.h"
#include "qpset_flatten.h"

namespace pcc {

namespace {

void
flatten(const RahtPredictionParams& rp, const QpSet& qs, bool rahtExtension,
        pccb200_raht_params& p, pccb200_qpset& q)
{
  p.prediction_enabled = rp.raht_prediction_enabled_flag;
  p.integer_haar = rp.integer_haar_enable_flag;
  p.prediction_threshold0 = rp.raht_prediction_threshold0;
  p.prediction_threshold1 = rp.raht_prediction_threshold1;
  p.subnode_prediction_enabled = rp.raht_subnode_prediction_enabled_flag;
  p.prediction_search_range = rp.raht_prediction_search_range;
  for (int i = 0; i < 19; i++)
    p.pred_weight_parent[i] = rp.predWeightParent[i];
  for (int i = 0; i < 12; i++)
    p.pred_weight_child[i] =
      i < int(rp.predWeightChild.size()) ? rp.predWeightChild[i] : 0;
  p.raht_extension = rahtExtension;

  flatten_qpset(qs, q);
}

// Qps is std::array<int, 2>: the per-point offsets are already a contiguous
// N x 2 int array; all-zero offsets (the CTC case) are passed as NULL
const int32_t*
qp_offsets(const Qps* pointQpOffsets, int n)
{
  static_assert(sizeof(Qps) == 2 * sizeof(int32_t), "Qps layout");
  const int32_t* flat = reinterpret_cast<const int32_t*>(pointQpOffsets);
  for (int i = 0; i < 2 * n; i++)
    if (flat[i])
      return flat;
  return nullptr;
}

void
check(int rc)
{
  if (rc != PCCB200_OK)
    throw std::runtime_error(std::string("pcc_attr_b200: ") + pccb200_last_error());
}

}  // namespace

void
regionAdaptiveHierarchicalTransform(
  const RahtPredictionParams& rahtPredParams,
  const QpSet& qpset,
  const Qps* pointQpOffsets,
  int64_t* mortonCode,
  int* attributes,
  const int attribCount,
  const int voxelCount,
  int* coefficients,
  const bool rahtExtension,
  AttributeInterPredParams& attrInterPredParams)
{
  if (attrInterPredParams.enableAttrInterPred)
    throw std::runtime_error("pcc_attr_b200: RAHT inter-frame prediction is not supported");
  pccb200_raht_params p;
  pccb200_qpset q;
  flatten(rahtPredParams, qpset, rahtExtension, p, q);
  check(pccb200_raht_forward(
    &p, &q, qp_offsets(pointQpOffsets, voxelCount), mortonCode, attributes,
    attribCount, voxelCount, coefficients));
}

void
regionAdaptiveHierarchicalInverseTransform(
  const RahtPredictionParams& rahtPredParams,
  const QpSet& qpset,
  const Qps* pointQpOffsets,
  int64_t* mortonCode,
  int* attributes,
  const int attribCount,
  const int voxelCount,
  int* coefficients,
  const bool rahtExtension,
  AttributeInterPredParams& attrInterPredParams)
{
  if (attrInterPredParams.enableAttrInterPred)
    throw std::runtime_error("pcc_attr_b200: RAHT inter-frame prediction is not supported");
  pccb200_raht_params p;
  pccb200_qpset q;
  flatten(rahtPredParams, qpset, rahtExtension, p, q);
  check(pccb200_raht_inverse(
    &p, &q, qp_offsets(pointQpOffsets, voxelCount), mortonCode, attributes,
    attribCount, voxelCount, coefficients));
}

}  // namespace pcc
