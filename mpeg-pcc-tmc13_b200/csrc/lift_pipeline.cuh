// lift_pipeline.cuh — the lifting attribute coder without its entropy coding
// (AttributeEncoder::encode{Colors,Reflectances}Lift,
// tmc3/AttributeEncoder.cpp:1379-1494,1543-1648, and the decoder's
// decode{Colors,Reflectances}Lift, tmc3/AttributeDecoder.cpp:678-857) as one
// executor-generic schedule: LoD build -> quantisation weights -> forward
// lifting -> last-component prediction + quantisation -> inverse lifting ->
// rounding, clip and write-back in point order.
#pragma once

#include "lifting.cuh"
#include "lod_pipeline.cuh"

namespace pccb200 {

// The attribute-independent part of a lifting call: levels of detail,
// predictors, quantisation weights (executor memory).  The reference keeps
// it across the attributes of a slice (AttributeEncoder::_lods,
// tmc3/AttributeEncoder.h:183; reuse rule AttributeLods::isReusable,
// tmc3/AttributeCommon.cpp:76-140).
struct LodState {
  int n;
  int numDetailLevels;
  pccb200_predictor* preds;  // n, predictor order
  uint32_t* idx;             // n, predictor order -> point index
  uint64_t* qw;              // n, quantisation weights
  uint32_t npl[PCCB200_MAX_LODS];
  int lodCount;
};

// fills st (preds / idx / qw must point to n entries each).  scal: scalable
// lifting, whose quantisation weights the encoder computes with (n, 0)
// (tmc3/AttributeEncoder.cpp:1390-1395) and the decoder with
// (geom_num_points, min_geom_node_size_log2) (tmc3/AttributeDecoder.cpp:692-697).
template<class Exec>
int
lod_state_build(Exec& ex, const pccb200_lod_params& lod, const int32_t* xyz, int n, LodState& st,
                bool withWeights = true, const pccb200_lod_scalable* scal = nullptr,
                bool decoder = false)
{
  st.n = n;
  st.numDetailLevels = scal ? kScalableLevels : lod.num_detail_levels;
  st.lodCount = 0;
  int rc = lod_run(ex, lod, xyz, n, st.preds, st.idx, st.npl, &st.lodCount, scal);
  if (rc != PCCB200_OK)
    return rc;
  // (the quantisation weights belong to the lifting transform; a caller that
  // may only need the predictors -- the predicting transform, whose coding loop
  // stays on the host -- asks for them later)
  if (!withWeights)
    return PCCB200_OK;
  if (scal) {
    const bool partial = decoder && scal->geom_num_points;
    return run_quant_weights_scalable(ex, st.npl, st.lodCount,
                                      uint64_t(partial ? scal->geom_num_points : n),
                                      decoder ? scal->min_geom_node_size_log2 : 0, n, st.qw);
  }
  return run_quant_weights(ex, st.preds, n, st.npl, st.lodCount, st.qw);
}

// One attribute set of a lifting call: what is coded per attribute on shared
// levels of detail.  attrsIn [n*A] (encoder) and attrsOut [n*A]
// (reconstruction): point order, executor memory; they may alias.  values
// [n*A]: coding order, executor memory (out when forward).  lcp: host array of
// PCCB200_MAX_LODS + 1 entries (computed when forward, read otherwise; used
// with A == 3 and lcpEnabled only).
constexpr int kLiftMaxSets = 4;

struct LiftSet {
  int A;          // 1 or 3
  int bitdepth;   // 1..16
  const pccb200_qpset* qpset;
  bool lcpEnabled;
  const int32_t* attrsIn;
  int32_t* attrsOut;
  int32_t* values;
  int8_t* lcp;
};

// 1..kLiftMaxSets attribute sets on prepared levels of detail (the case where
// the reference reuses _lods for the next attribute).  The sets' components
// are gathered side by side into one row per point (SA = the sum of their A),
// so the forward and inverse lifting passes run once for all of them, with the
// launches of one set; gather, quantisation (own QpSet, own last-component
// prediction) and the clipped write-back are launched once per set.  Each
// set's results are bit-identical to a call with that set alone.  qpoIn
// [n*2] or null: point order, executor memory, applies to every set.
template<class Exec>
int
attr_lift_on_lods(Exec& ex, bool forward, const LodState& st, const int32_t* qpoIn, int numSets,
                  const LiftSet* sets)
{
  if (numSets < 1 || numSets > kLiftMaxSets)
    return PCCB200_ERR_INVALID_ARG;
  int SA = 0;
  for (int s = 0; s < numSets; s++) {
    if (sets[s].A != 1 && sets[s].A != 3)
      return PCCB200_ERR_INVALID_ARG;
    SA += sets[s].A;
  }
  const int n = st.n;
  int64_t* coef = ex.template alloc<int64_t>(size_t(n) * SA);
  int32_t* qpo = nullptr;
  if (qpoIn) {
    qpo = ex.template alloc<int32_t>(size_t(n) * 2);
    ex.foreach(n, GatherQpoFn{qpoIn, st.idx, qpo});
  }
  int rc;
  if (forward) {
    for (int s = 0, off = 0; s < numSets; off += sets[s].A, s++)
      ex.foreach(n, GatherAttrShiftFn{sets[s].attrsIn, st.idx, sets[s].A, SA, off, coef});
    rc = run_lift(ex, true, st.preds, st.qw, n, st.npl, st.lodCount, coef, SA);
    if (rc != PCCB200_OK)
      return rc;
  }
  for (int s = 0, off = 0; s < numSets; off += sets[s].A, s++) {
    const LiftSet& t = sets[s];
    rc = run_lift_quant(ex, forward, *t.qpset, qpo, st.qw, n, st.npl, st.lodCount,
                        st.numDetailLevels, coef, SA, off, t.A, t.lcpEnabled, t.lcp, t.values);
    if (rc != PCCB200_OK)
      return rc;
  }
  rc = run_lift(ex, false, st.preds, st.qw, n, st.npl, st.lodCount, coef, SA);
  if (rc != PCCB200_OK)
    return rc;
  for (int s = 0, off = 0; s < numSets; off += sets[s].A, s++)
    ex.foreach(n, ScatterReconFn{coef, st.idx, sets[s].A, SA, off, (1 << sets[s].bitdepth) - 1,
                                 sets[s].attrsOut});
  return PCCB200_OK;
}

// One attribute on prepared levels of detail.  attrsIn [n*A] (encoder),
// qpoIn [n*2] or null: point order, executor memory.  values [n*A]: coding
// order (out when forward).  attrsOut [n*A]: reconstruction in point order.
// lcp: host array of PCCB200_MAX_LODS + 1 entries.
template<class Exec>
int
attr_lift_on_lods(Exec& ex, bool forward, const LodState& st, const pccb200_qpset& qpset,
                  bool lcpEnabled, const int32_t* qpoIn, const int32_t* attrsIn,
                  int32_t* attrsOut, int A, int bitdepth, int32_t* values, int8_t* lcp)
{
  const LiftSet set{A, bitdepth, &qpset, lcpEnabled, attrsIn, attrsOut, values, lcp};
  return attr_lift_on_lods(ex, forward, st, qpoIn, 1, &set);
}

// Levels of detail of xyz [n*3] (executor memory), then attr_lift_on_lods.
// scal: scalable lifting, or null.
template<class Exec>
int
attr_lift_run(Exec& ex, bool forward, const pccb200_lod_params& lod, const int32_t* qpoIn,
              const int32_t* xyz, int n, int numSets, const LiftSet* sets,
              const pccb200_lod_scalable* scal = nullptr)
{
  LodState st;
  st.preds = ex.template alloc<pccb200_predictor>(n);
  st.idx = ex.template alloc<uint32_t>(n);
  st.qw = ex.template alloc<uint64_t>(n);
  int rc = lod_state_build(ex, lod, xyz, n, st, true, scal, !forward);
  if (rc != PCCB200_OK)
    return rc;
  return attr_lift_on_lods(ex, forward, st, qpoIn, numSets, sets);
}

// xyz [n*3], attrsIn [n*A] (encoder), qpoIn [n*2] or null: point order,
// executor memory.  values [n*A]: coding order (out when forward).
// attrsOut [n*A]: reconstruction in point order.  lcp: host array of
// PCCB200_MAX_LODS + 1 entries.
template<class Exec>
int
attr_lift_run(Exec& ex, bool forward, const pccb200_lod_params& lod, const pccb200_qpset& qpset,
              bool lcpEnabled, const int32_t* qpoIn, const int32_t* xyz, const int32_t* attrsIn,
              int32_t* attrsOut, int A, int n, int bitdepth, int32_t* values, int8_t* lcp)
{
  const LiftSet set{A, bitdepth, &qpset, lcpEnabled, attrsIn, attrsOut, values, lcp};
  return attr_lift_run(ex, forward, lod, qpoIn, xyz, n, 1, &set);
}

}  // namespace pccb200
