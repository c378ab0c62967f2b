// pred_decode.cuh — the predicting transform's decoder without its entropy
// decoding (AttributeDecoder::decode{Reflectances,Colors}Pred,
// tmc3/AttributeDecoder.cpp:328-391,446-523).
//
// The entropy decoding of the reference's loop never reads a reconstruction,
// so the caller hands over the decoded values in coding order.  What is left
// is closed-loop DPCM: a point's eligibility for a direct predictor, its
// prediction and hence its reconstruction read the reconstructions of its
// (at most three) neighbours, whose predictor indexes are below its own.
// Decoding is therefore a dataflow over a DAG known before any value is read:
// on the device, one k_warp_flow launch (exec_cuda.cuh) over the chains of a
// gang claims points in predictor order, 32 per warp ticket, and every point
// publishes its reconstruction with one 64-bit store into a slot that holds 0
// (no published record has that value) until then.
#pragma once

#include <vector>

#include "lifting.cuh"

namespace pccb200 {

// one attribute set of one unit: one chain of the dataflow
struct PredChain {
  const pccb200_predictor* preds;  // n, predictor order
  const uint64_t* qw;              // n, fixed-weight quantisation weights
  const int32_t* qpo;              // n * 2 in predictor order, or null
  const int32_t* values;           // n * A, coding order
  unsigned long long* slots;       // n records, 0 until published
  unsigned long long* ticket;
  int64_t n;
  int A;                           // 1 (reflectance) or 3 (colour)
  int32_t clipMax;                 // 2^bitdepth - 1
  int32_t threshold;               // adaptivePredictionThreshold (hls.h:808-811)
  int maxNumDirect;                // max_num_direct_predictors
  int avgDisabled;                 // direct_avg_predictor_disabled_flag
  int icpEnabled;                  // inter_component_prediction_enabled_flag
  int numLayers;
  LayerQp layers[PCCB200_MAX_QP_LAYERS];
  LodTable lt;                     // the strictly increasing prefix of numPointsInLod
  int8_t icp[PCCB200_MAX_LODS][3]; // icpCoeffs[lod], zero when absent
};

// a published record: bit 63 set, the clipped value(s) in 16-bit fields
constexpr unsigned long long kPredReady = 1ull << 63;

PCC_HD unsigned long long
pred_slot_load(const unsigned long long* p)
{
#if defined(__CUDA_ARCH__)
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
#else
  return *p;
#endif
}

PCC_HD void
pred_slot_store(unsigned long long* p, unsigned long long v)
{
#if defined(__CUDA_ARCH__)
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
  *p = v;
#endif
}

PCC_HD int32_t
pred_abs(int32_t v)
{
  return v < 0 ? -v : v;
}

// The reference's per-point decode step for predictor i.  Returns false, and
// changes nothing, while a neighbour's reconstruction is not published.
struct PredDecodeFn {
  const PredChain* c;
  unsigned long long* ticket;  // of the dataflow launch (c->ticket)
  PCC_HD int64_t size() const { return c->n; }
  PCC_HD bool operator()(int64_t i) const
  {
    const PredChain& ch = *c;
    const pccb200_predictor& p = ch.preds[i];
    const uint32_t nc = p.neighbor_count;
    const int A = ch.A;
    unsigned long long rec[3] = {0, 0, 0};
    for (uint32_t j = 0; j < nc; j++) {
      rec[j] = pred_slot_load(&ch.slots[p.predictor_index[j]]);
      if (!(rec[j] & kPredReady))
        return false;
    }
    auto comp = [&](uint32_t j, int k) -> int64_t { return int64_t((rec[j] >> (16 * k)) & 0xffff); };

    // quantLayer and the ICP level advance at each boundary of numPointsInLod
    // (AttributeDecoder.cpp:350-352,473-475,485-486)
    const int lod = ch.lt.lod_of(i);
    const int layer = lod < ch.numLayers - 1 ? lod : ch.numLayers - 1;
    Quantizer q[2];
    make_quantizers(ch.layers[layer], ch.qpo ? ch.qpo[2 * i] : 0, ch.qpo ? ch.qpo[2 * i + 1] : 0,
                    q);
    int32_t v[3] = {0, 0, 0};
    for (int k = 0; k < A; k++)
      v[k] = ch.values[i * A + k];

    // predModeEligible{Color,Refl} (AttributeCommon.cpp:145-210) on the
    // reconstructed neighbours, then decodePredMode{Color,Refl}
    // (AttributeDecoder.cpp:289-323,396-441)
    int predMode = 0;
    if (nc > 1 && ch.maxNumDirect) {
      int64_t maxDiff = 0;
      for (int k = 0; k < A; k++) {
        int64_t lo = comp(0, k), hi = lo;
        for (uint32_t j = 1; j < nc; j++) {
          const int64_t x = comp(j, k);
          lo = x < lo ? x : lo;
          hi = x > hi ? x : hi;
        }
        maxDiff = hi - lo > maxDiff ? hi - lo : maxDiff;
      }
      if (maxDiff >= ch.threshold) {
        const int maxcand = ch.maxNumDirect + !ch.avgDisabled;
        int mode = 0;
        if (A == 3) {
          const int32_t s1 = v[1] < 0 ? -1 : 1, s2 = v[2] < 0 ? -1 : 1;
          const int32_t a1 = pred_abs(v[1]), a2 = pred_abs(v[2]);
          if (maxcand == 4) {
            v[1] = s1 * (a1 >> 1);
            v[2] = s2 * (a2 >> 1);
            mode = ((a1 & 1) << 1) + (a2 & 1);
          } else if (maxcand == 3) {
            v[1] = s1 * (a1 >> 1);
            mode = a1 & 1;
            if (mode) {
              v[2] = s2 * (a2 >> 1);
              mode += a2 & 1;
            }
          } else if (maxcand == 2) {
            v[1] = s1 * (a1 >> 1);
            mode = a1 & 1;
          }
        } else {
          const int32_t s = v[0] < 0 ? -1 : 1;
          int32_t a = pred_abs(v[0]);
          if (maxcand == 4) {
            mode = a & 3;
            v[0] = s * (a >> 2);
          } else if (maxcand == 3) {
            mode = a & 1;
            a >>= 1;
            if (mode > 0) {
              mode += a & 1;
              a >>= 1;
            }
            v[0] = s * a;
          } else if (maxcand == 2) {
            mode = a & 1;
            v[0] = s * (a >> 1);
          }
        }
        predMode = mode + ch.avgDisabled;
      }
    }

    // predictColor / predictReflectance (PCCTMC3Common.h:526-587): a colour
    // weight is taken as uint32 and the colour comes back as Vec3<attr_t>,
    // i.e. truncated to 16 bits; a reflectance product is 64-bit
    int64_t pred[3] = {0, 0, 0};
    if (uint32_t(predMode) > nc) {
      /* prediction 0 */
    } else if (predMode > 0) {
      for (int k = 0; k < A; k++)
        pred[k] = comp(uint32_t(predMode - 1), k);
    } else {
      for (int k = 0; k < A; k++) {
        int64_t acc = 0;
        for (uint32_t j = 0; j < nc; j++)
          acc += A == 3 ? int64_t(uint32_t(p.weight[j] * uint32_t(comp(j, k))))
                        : int64_t(uint64_t(p.weight[j]) * uint64_t(comp(j, k)));
        pred[k] = div_exp2_round_half_inf(acc, 8);
        if (A == 3)
          pred[k] = int64_t(uint16_t(pred[k]));
      }
    }

    unsigned long long out = kPredReady;
    int64_t residual0 = 0;
    for (int k = 0; k < A; k++) {
      const Quantizer& qk = q[k < 1 ? k : 1];
      const int64_t qStep = qk.step;
      const int64_t qwi = int64_t(ch.qw[i]);
      const int64_t weight = (qwi < qStep ? qwi : qStep) >> 8;
      const int64_t residual = div_exp2_round_half_up(qk.scale(v[k]), 8) / weight;
      int64_t recon = pred[k] + residual;
      if (A == 3)
        recon += (int64_t(ch.icp[lod][k]) * residual0 + 2) >> 2;
      recon = recon < 0 ? 0 : (recon > ch.clipMax ? ch.clipMax : recon);
      out |= (unsigned long long)recon << (16 * k);
      if (!k && ch.icpEnabled)
        residual0 = residual;
    }
    pred_slot_store(&ch.slots[i], out);
    return true;
  }
};

// the clipped reconstruction of predictor i to its point: out[idx[i]][k]
struct PredScatterFn {
  const unsigned long long* slots;
  const uint32_t* idx;
  int A;
  int32_t* out;
  PCC_HD void operator()(int64_t i) const
  {
    const unsigned long long r = slots[i];
    for (int k = 0; k < A; k++)
      out[size_t(idx[i]) * A + k] = int32_t((r >> (16 * k)) & 0xffff);
  }
};

// flag: a predictor is malformed (more than three neighbours) or references
// a predictor index not below its own.  Such a reference would leave a poll
// of the decoding dataflow waiting forever, so it is refused before any launch.
struct PredCheckFn {
  const pccb200_predictor* preds;
  int* flag;
  PCC_HD void operator()(int64_t i) const
  {
    const pccb200_predictor& p = preds[i];
    if (p.neighbor_count > 3) {
      atomic_or_i32(flag, 1);
      return;
    }
    for (uint32_t j = 0; j < p.neighbor_count; j++)
      if (int64_t(p.predictor_index[j]) >= i)
        atomic_or_i32(flag, 1);
  }
};

// hChains: the table on the host; dChains: the same in executor memory.
// An executor with a dataflow launch (the device) runs every chain in one
// k_warp_flow launch; any other runs the chains one after the other, each in
// predictor order (an order in which every neighbour is published before it
// is read).
template<class Exec>
auto
pred_decode_chains(Exec& ex, const PredChain* hChains, const PredChain* dChains, int numChains,
                   int) -> decltype(ex.flow((const PredDecodeFn*)nullptr,
                                            (const PredDecodeFn*)nullptr, 0), void())
{
  std::vector<PredDecodeFn> fns(numChains);
  for (int c = 0; c < numChains; c++)
    fns[c] = PredDecodeFn{&dChains[c], hChains[c].ticket};
  PredDecodeFn* dFns = ex.template alloc<PredDecodeFn>(size_t(numChains));
  ex.upload(dFns, fns.data(), fns.size() * sizeof(PredDecodeFn));
  // (the grid reads size() from the host copy of each chain)
  std::vector<PredDecodeFn> hFns(numChains);
  for (int c = 0; c < numChains; c++)
    hFns[c] = PredDecodeFn{&hChains[c], hChains[c].ticket};
  ex.flow(hFns.data(), dFns, numChains);
}

template<class Exec>
void
pred_decode_chains(Exec& ex, const PredChain* hChains, const PredChain*, int numChains, long)
{
  for (int c = 0; c < numChains; c++)
    ex.foreach(hChains[c].n, PredDecodeFn{&hChains[c], hChains[c].ticket});
}

}  // namespace pccb200
