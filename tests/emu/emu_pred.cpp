// emu_pred.cpp — TEST INFRASTRUCTURE ONLY: the predicting-transform decoder
// (pred_pipeline.cuh, pred_decode.cuh) and the counter-driven quantisation
// weights (lifting.cuh) compiled for the host and run as loops (see
// exec_host.h).  Built by tests/test_pred_decode_host.py into a temporary
// directory.
#include <algorithm>
#include <random>
#include <vector>

#include "exec_host.h"
#include "pred_pipeline.cuh"

namespace {

// runs f(t) for t in [0, n) in a seeded random order of attempts until every
// item has returned true: any order a dataflow launch may take
template<class F>
int64_t
random_schedule(int64_t n, const F& f, unsigned seed)
{
  std::mt19937 rng(seed);
  std::vector<int64_t> pending(n);
  for (int64_t t = 0; t < n; t++)
    pending[t] = t;
  int64_t refused = 0;
  while (!pending.empty()) {
    // a window of the lowest pending tickets, as warps hold them
    const size_t w = std::min<size_t>(pending.size(), 64);
    std::uniform_int_distribution<size_t> pick(0, w - 1);
    const size_t k = pick(rng);
    if (f(pending[k]))
      pending.erase(pending.begin() + k);
    else
      refused++;
  }
  return refused;
}

}  // namespace

// The product's pipeline on the host: levels of detail given (predictor
// order), one set.  Returns the status of attr_pred_decode_on_lods.
extern "C" int
emu_pred_decode(const pccb200_predictor* preds, const uint32_t* indexes, int n, const uint32_t* npl,
                int lodCount, const pccb200_qpset* qs, const pccb200_pred_params* pp,
                const int32_t qnw[3], const int32_t* qpo, const int8_t* icp, const int32_t* values,
                int A, int bitdepth, int32_t* out)
{
  HostExec ex;
  pccb200::LodState st;
  st.n = n;
  st.numDetailLevels = lodCount;
  st.preds = const_cast<pccb200_predictor*>(preds);
  st.idx = const_cast<uint32_t*>(indexes);
  st.qw = nullptr;
  st.lodCount = lodCount;
  for (int l = 0; l < lodCount; l++)
    st.npl[l] = npl[l];
  pccb200::PredUnit u = {};
  u.st = &st;
  u.qpo = qpo;
  for (int k = 0; k < 3; k++)
    u.quantNeighWeight[k] = qnw[k];
  u.numSets = 1;
  u.sets[0] = pccb200::PredSet{A, bitdepth, qs, *pp, values, icp, out};
  return pccb200::attr_pred_decode_on_lods(ex, 1, &u);
}

// PredDecodeFn alone, driven in a random order of attempts: qw given; the
// slots and decoded values in predictor order (out[i * A + k]).  Returns the
// number of refused attempts.
extern "C" int64_t
emu_pred_decode_sched(const pccb200_predictor* preds, const uint64_t* qw, int n, const uint32_t* npl,
                      int lodCount, const pccb200_qpset* qs, const pccb200_pred_params* pp,
                      const int32_t* qpoPred, const int8_t* icp, const int32_t* values, int A,
                      int bitdepth, unsigned seed, int32_t* out)
{
  std::vector<unsigned long long> slots(n ? n : 1, 0);
  unsigned long long ticket = 0;
  pccb200::PredChain ch = {};
  ch.preds = preds;
  ch.qw = qw;
  ch.qpo = qpoPred;
  ch.values = values;
  ch.slots = slots.data();
  ch.ticket = &ticket;
  ch.n = n;
  ch.A = A;
  ch.clipMax = (1 << bitdepth) - 1;
  ch.threshold = pp->adaptive_prediction_threshold << std::max(0, bitdepth - 8);
  ch.maxNumDirect = pp->max_num_direct_predictors;
  ch.avgDisabled = pp->direct_avg_predictor_disabled;
  ch.icpEnabled = pp->icp_enabled;
  ch.numLayers = qs->num_layers;
  for (int l = 0; l < qs->num_layers; l++)
    ch.layers[l] = pccb200::LayerQp{qs->layers[l][0], qs->layers[l][1], qs->max_qp,
                                    qs->fixed_point_qp_offset};
  ch.lt.lodCount = 0;
  while (ch.lt.lodCount < lodCount
         && npl[ch.lt.lodCount] > (ch.lt.lodCount ? npl[ch.lt.lodCount - 1] : 0u)) {
    ch.lt.npl[ch.lt.lodCount] = npl[ch.lt.lodCount];
    ch.lt.lodCount++;
  }
  for (int l = 0; l < PCCB200_MAX_LODS; l++)
    for (int k = 0; k < 3; k++)
      ch.icp[l][k] = icp ? icp[3 * l + k] : 0;
  const int64_t refused = random_schedule(n, pccb200::PredDecodeFn{&ch}, seed);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < A; k++)
      out[size_t(i) * A + k] = int32_t((slots[i] >> (16 * k)) & 0xffff);
  return refused;
}

// run_quant_weights with the fixed neighbour weights, where a level that
// references itself runs QwReferrerCountFn + QwFlowFn in a random order of
// attempts instead of the host's sequential walk.  Returns the number of
// refused attempts, or -1 for malformed levels.
extern "C" int64_t
emu_quant_weights_flow(const pccb200_predictor* preds, int n, const uint32_t* npl, int lodCount,
                       const int32_t qnw[3], unsigned seed, uint64_t* qw)
{
  HostExec ex;
  const pccb200::NeighWeights nw{{qnw[0], qnw[1], qnw[2]}, 1};
  std::vector<int> cnt(n ? n : 1, 0);
  ex.foreach(n, pccb200::FillU64Fn{qw, uint64_t(1) << 8});
  int64_t refused = 0;
  for (int l = lodCount - 1; l >= 0; l--) {
    const int64_t s = l ? npl[l - 1] : 0, e = npl[l];
    int flag = 0;
    ex.foreach(e - s, pccb200::LodCheckFn{preds, s, &flag, n});
    if (flag & 6)
      return -1;
    if (!flag) {
      ex.foreach(e - s, pccb200::QuantWeightLodFn{preds, qw, s, nw});
      continue;
    }
    std::fill(cnt.begin(), cnt.end(), 0);
    ex.foreach(e - s, pccb200::QwReferrerCountFn{preds, cnt.data(), s});
    refused += random_schedule(e - s, pccb200::QwFlowFn{preds, qw, cnt.data(), s, e, nw}, seed + l);
    for (int64_t i = 0; i < e - s; i++)
      if (cnt[i])
        return -1;
  }
  return refused;
}

// the product's run_quant_weights on the host (QuantWeightSeqFn for a level
// that references itself)
extern "C" int
emu_quant_weights_fixed(const pccb200_predictor* preds, int n, const uint32_t* npl, int lodCount,
                        const int32_t qnw[3], uint64_t* qw)
{
  HostExec ex;
  return pccb200::run_quant_weights(ex, preds, n, npl, lodCount, qw, qnw);
}
