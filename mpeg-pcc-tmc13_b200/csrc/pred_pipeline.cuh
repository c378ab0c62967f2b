// pred_pipeline.cuh — the predicting-transform decoder on prepared levels of
// detail, for a gang of units: fixed-weight quantisation weights
// (computeQuantizationWeights with quant_neigh_weight,
// tmc3/AttributeDecoder.cpp:343-345,464-466), gathered qp offsets, seeded
// slots, one k_warp_flow dataflow over every attribute set of every unit,
// and the clipped values scattered to point order.
#pragma once

#include "lift_pipeline.cuh"
#include "pred_decode.cuh"

namespace pccb200 {

constexpr int kPredMaxSets = 4;

// one attribute set of a unit.  values [n*A]: coding order, attrsOut [n*A]:
// point order, executor memory.  icp: host row of PCCB200_MAX_LODS triplets
// (icpCoeffs per level of detail), or null for none.
struct PredSet {
  int A;         // 1 or 3
  int bitdepth;  // 1..16
  const pccb200_qpset* qpset;
  pccb200_pred_params pp;
  const int32_t* values;
  const int8_t* icp;
  int32_t* attrsOut;
};

// one unit: its levels of detail, qp offsets [n*2] in point order (executor
// memory) or null, quant_neigh_weight, and 1..kPredMaxSets sets
struct PredUnit {
  const LodState* st;
  const int32_t* qpo;
  int32_t quantNeighWeight[3];
  int numSets;
  PredSet sets[kPredMaxSets];
};

// PCCB200_ERR_INVALID_ARG, before any dataflow launch, if a predictor of a
// unit references a predictor index not below its own, or if its levels of
// detail are malformed (*badUnit names the unit, *why the cause)
template<class Exec>
int
attr_pred_decode_on_lods(Exec& ex, int numUnits, const PredUnit* units, int* badUnit = nullptr,
                         const char** why = nullptr)
{
  if (numUnits < 1)
    return PCCB200_ERR_INVALID_ARG;
  int numChains = 0;
  for (int u = 0; u < numUnits; u++) {
    if (units[u].numSets < 1 || units[u].numSets > kPredMaxSets)
      return PCCB200_ERR_INVALID_ARG;
    for (int s = 0; s < units[u].numSets; s++) {
      const PredSet& t = units[u].sets[s];
      if ((t.A != 1 && t.A != 3) || t.bitdepth < 1 || t.bitdepth > 16 || t.qpset->num_layers < 1
          || t.qpset->num_layers > PCCB200_MAX_QP_LAYERS)
        return PCCB200_ERR_INVALID_ARG;
    }
    numChains += units[u].numSets;
  }
  ex.phase(5);
  int* dFlags = ex.template alloc<int>(size_t(numUnits));
  ex.zero(dFlags, size_t(numUnits) * sizeof(int));
  for (int u = 0; u < numUnits; u++)
    ex.foreach(units[u].st->n, PredCheckFn{units[u].st->preds, dFlags + u});
  std::vector<int> flags(numUnits);
  ex.download(flags.data(), dFlags, flags.size() * sizeof(int));
  for (int u = 0; u < numUnits; u++)
    if (flags[u]) {
      if (badUnit)
        *badUnit = u;
      if (why)
        *why = "a predictor references a predictor index not below its own, or has more than "
               "three neighbours";
      return PCCB200_ERR_INVALID_ARG;
    }

  std::vector<PredChain> chains(numChains);
  unsigned long long* tickets = ex.template alloc<unsigned long long>(size_t(numChains));
  ex.zero(tickets, size_t(numChains) * sizeof(unsigned long long));
  for (int u = 0, c = 0; u < numUnits; u++) {
    const PredUnit& pu = units[u];
    const LodState& st = *pu.st;
    const int64_t n = st.n;
    uint64_t* qw = ex.template alloc<uint64_t>(size_t(n));
    int rc = run_quant_weights(ex, st.preds, n, st.npl, st.lodCount, qw, pu.quantNeighWeight);
    if (rc != PCCB200_OK) {
      if (badUnit)
        *badUnit = u;
      if (why)
        *why = "numPointsInLod does not partition [0, n), or a neighbour lies outside [0, n)";
      return rc;
    }
    int32_t* qpo = nullptr;
    if (pu.qpo) {
      qpo = ex.template alloc<int32_t>(size_t(n) * 2);
      ex.foreach(n, GatherQpoFn{pu.qpo, st.idx, qpo});
    }
    // the strictly increasing prefix of numPointsInLod takes effect (see
    // run_lift_quant: the reference's `if (i == npl[lod]) lod++`)
    LodTable lt;
    lt.lodCount = 0;
    while (lt.lodCount < st.lodCount
           && st.npl[lt.lodCount] > (lt.lodCount ? st.npl[lt.lodCount - 1] : 0u)) {
      lt.npl[lt.lodCount] = st.npl[lt.lodCount];
      lt.lodCount++;
    }
    for (int s = 0; s < pu.numSets; s++, c++) {
      const PredSet& t = pu.sets[s];
      PredChain& ch = chains[c];
      ch.preds = st.preds;
      ch.qw = qw;
      ch.qpo = qpo;
      ch.values = t.values;
      ch.slots = ex.template alloc<unsigned long long>(size_t(n));
      ex.zero(ch.slots, size_t(n) * sizeof(unsigned long long));
      ch.ticket = tickets + c;
      ch.n = n;
      ch.A = t.A;
      ch.clipMax = (int32_t(1) << t.bitdepth) - 1;
      ch.threshold = t.pp.adaptive_prediction_threshold << (t.bitdepth > 8 ? t.bitdepth - 8 : 0);
      ch.maxNumDirect = t.pp.max_num_direct_predictors;
      ch.avgDisabled = t.pp.direct_avg_predictor_disabled ? 1 : 0;
      ch.icpEnabled = t.pp.icp_enabled ? 1 : 0;
      ch.numLayers = t.qpset->num_layers;
      for (int l = 0; l < ch.numLayers; l++) {
        ch.layers[l].luma = t.qpset->layers[l][0];
        ch.layers[l].chromaOffset = t.qpset->layers[l][1];
        ch.layers[l].maxQp = t.qpset->max_qp;
        ch.layers[l].fixedPointQpOffset = t.qpset->fixed_point_qp_offset;
      }
      ch.lt = lt;
      for (int l = 0; l < PCCB200_MAX_LODS; l++)
        for (int k = 0; k < 3; k++)
          ch.icp[l][k] = t.icp ? t.icp[3 * l + k] : 0;
    }
  }
  PredChain* dChains = ex.template alloc<PredChain>(size_t(numChains));
  ex.upload(dChains, chains.data(), chains.size() * sizeof(PredChain));
  pred_decode_chains(ex, chains.data(), dChains, numChains, 0);
  for (int u = 0, c = 0; u < numUnits; u++)
    for (int s = 0; s < units[u].numSets; s++, c++)
      ex.foreach(units[u].st->n, PredScatterFn{chains[c].slots, units[u].st->idx,
                                               units[u].sets[s].A, units[u].sets[s].attrsOut});
  return PCCB200_OK;
}

}  // namespace pccb200
