// lifting.cuh — the lifting transform's data-parallel passes.
//
//   quantisation weights  PCCComputeQuantizationWeights  tmc3/PCCTMC3Common.h:828-854
//   prediction step       PCCLiftPredict                 tmc3/PCCTMC3Common.h:716-770
//   update step           PCCLiftUpdate                  tmc3/PCCTMC3Common.h:774-824
//   LoD loops             tmc3/AttributeEncoder.cpp:1408-1415 (forward),
//                         tmc3/AttributeEncoder.cpp:1476-1482 (inverse)
//
// The reference walks predictors one by one; because the lifting transform
// only ever predicts from strictly coarser levels of detail
// (tmc3/encoder.cpp:777-780), every LoD is one data-parallel launch, and the
// scatter-adds of the update step and of the quantisation weights are 64-bit
// integer atomics: addition modulo 2^64 is order independent, so the results
// are bit-identical to the sequential walk.  A predictor that references its
// own LoD is reported through an error word; the quantisation weights of such
// a level are a counter-driven dataflow on the device (QwFlowFn).
#pragma once

#include <vector>

#include "pcc_arith.cuh"
#include "raht_core.cuh"

namespace pccb200 {

PCC_HD void
atomic_add_u64(uint64_t* p, uint64_t v)
{
#if defined(__CUDA_ARCH__)
  atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
#else
  *p += v;
#endif
}

struct FillU64Fn {
  uint64_t* p;
  uint64_t v;
  PCC_HD void operator()(int64_t i) const { p[i] = v; }
};

// flag bit 0: a predictor in [start, start + n) references an index >= start
// (its own level of detail); bit 1: a predictor is malformed (more than three
// neighbours, or an index outside [0, total)); bit 2 (with bit 0): it
// references an index not below its own
struct LodCheckFn {
  const pccb200_predictor* preds;
  int64_t start;
  int* flag;
  int64_t total;
  PCC_HD void operator()(int64_t i) const
  {
    const pccb200_predictor& p = preds[start + i];
    if (p.neighbor_count > 3) {
      atomic_or_i32(flag, 2);
      return;
    }
    for (uint32_t j = 0; j < p.neighbor_count; j++) {
      if (int64_t(p.predictor_index[j]) >= total)
        atomic_or_i32(flag, 2);
      else if (int64_t(p.predictor_index[j]) >= start + i)
        atomic_or_i32(flag, 5);
      else if (int64_t(p.predictor_index[j]) >= start)
        atomic_or_i32(flag, 1);
    }
  }
};

PCC_HD int
atomic_add_old_i32(int* p, int v)
{
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  const int old = *p;
  *p += v;
  return old;
#endif
}

// levels of detail made by the caller (pccb200_lod_import), entry i of total:
// flag bit 0: indexes is not a permutation of [0, total) (an entry out of
// range, or one met twice; seen: total zeroed counters); bit 1: a predictor is
// malformed, as in LodCheckFn.  Both would turn the lifting gathers and
// scatters into out-of-bounds or racing accesses.
struct LodImportCheckFn {
  const pccb200_predictor* preds;
  const uint32_t* indexes;
  int* seen;
  int* flag;
  int64_t total;
  PCC_HD void operator()(int64_t i) const
  {
    const int64_t k = indexes[i];
    if (k >= total || atomic_add_old_i32(&seen[k], 1) != 0)
      atomic_or_i32(flag, 1);
    const pccb200_predictor& p = preds[i];
    if (p.neighbor_count > 3) {
      atomic_or_i32(flag, 2);
      return;
    }
    for (uint32_t j = 0; j < p.neighbor_count; j++)
      if (int64_t(p.predictor_index[j]) >= total)
        atomic_or_i32(flag, 2);
  }
};

// neighbour weight j of a predictor: its own (lifting, PCCTMC3Common.h:828-854)
// or the fixed per-slot weight of the predicting transform
// (computeQuantizationWeights, PCCTMC3Common.h:895-921)
struct NeighWeights {
  int32_t fixed[3];
  int useFixed;
  PCC_HD uint64_t of(const pccb200_predictor& p, uint32_t j) const
  {
    return useFixed ? uint64_t(int64_t(fixed[j])) : uint64_t(p.weight[j]);
  }
};

struct QuantWeightLodFn {
  const pccb200_predictor* preds;
  uint64_t* qw;
  int64_t start;
  NeighWeights nw;
  PCC_HD void operator()(int64_t i) const
  {
    const pccb200_predictor& p = preds[start + i];
    const uint64_t w = qw[start + i];
    for (uint32_t j = 0; j < p.neighbor_count; j++)
      atomic_add_u64(&qw[p.predictor_index[j]], div_exp2_round_half_inf_u(nw.of(p, j) * w, 8));
  }
};

// sequential walk of a range, last to first (used when a LoD references itself)
struct QuantWeightSeqFn {
  const pccb200_predictor* preds;
  uint64_t* qw;
  int64_t start, end;
  NeighWeights nw;
  PCC_HD void operator()(int64_t) const
  {
    for (int64_t i = end - 1; i >= start; i--) {
      const pccb200_predictor& p = preds[i];
      const uint64_t w = qw[i];
      for (uint32_t j = 0; j < p.neighbor_count; j++)
        qw[p.predictor_index[j]] += div_exp2_round_half_inf_u(nw.of(p, j) * w, 8);
    }
  }
};

// The same walk of a level [s, e) that references itself, as a dataflow over
// the level: cnt[i - s] counts the referrers of predictor i inside the level
// (QwReferrerCountFn).  Ticket t is predictor e - 1 - t.  Once its counter is
// 0, every contribution to its weight has been added (the referrers of a
// predictor have higher indexes); it adds its own to each neighbour, then --
// after a release fence -- decrements the counters of the neighbours inside
// the level.  Each contribution depends on a final weight only, and uint64
// addition commutes, so the weights equal QuantWeightSeqFn's bit for bit.
struct QwReferrerCountFn {
  const pccb200_predictor* preds;
  int* cnt;
  int64_t start;
  PCC_HD void operator()(int64_t i) const
  {
    const pccb200_predictor& p = preds[start + i];
    for (uint32_t j = 0; j < p.neighbor_count; j++)
      if (int64_t(p.predictor_index[j]) >= start)
        atomic_add_old_i32(&cnt[p.predictor_index[j] - start], 1);
  }
};

struct QwFlowFn {
  const pccb200_predictor* preds;
  uint64_t* qw;
  int* cnt;
  int64_t start, end;
  NeighWeights nw;
  unsigned long long* ticket;  // of the dataflow launch
  PCC_HD int64_t size() const { return end - start; }
  // false while a referrer of the predictor has not run yet
  PCC_HD bool operator()(int64_t t) const
  {
    const int64_t i = end - 1 - t;
#if defined(__CUDA_ARCH__)
    int c;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(c) : "l"(cnt + (i - start)) : "memory");
    if (c)
      return false;
    __threadfence();
    unsigned long long w;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(qw + i) : "memory");
#else
    if (cnt[i - start])
      return false;
    const uint64_t w = qw[i];
#endif
    const pccb200_predictor& p = preds[i];
    for (uint32_t j = 0; j < p.neighbor_count; j++)
      atomic_add_u64(&qw[p.predictor_index[j]], div_exp2_round_half_inf_u(nw.of(p, j) * w, 8));
#if defined(__CUDA_ARCH__)
    __threadfence();
#endif
    for (uint32_t j = 0; j < p.neighbor_count; j++)
      if (int64_t(p.predictor_index[j]) >= start)
        atomic_add_old_i32(&cnt[p.predictor_index[j] - start], -1);
    return true;
  }
};

// A level that references itself: the counter-driven QwFlowFn on an executor
// with a dataflow launch (the device), QuantWeightSeqFn in one thread on any
// other (the host emulation, where it is the check of the dataflow).
template<class Exec>
auto
quant_weights_self(Exec& ex, QwFlowFn f, int) -> decltype(ex.flow(&f, &f, 1), void())
{
  ex.zero(f.cnt, size_t(f.end - f.start) * sizeof(int));
  ex.foreach(f.end - f.start, QwReferrerCountFn{f.preds, f.cnt, f.start});
  f.ticket = ex.template alloc<unsigned long long>(1);
  ex.zero(f.ticket, sizeof(unsigned long long));
  QwFlowFn* d = ex.template alloc<QwFlowFn>(1);
  ex.upload(d, &f, sizeof(f));
  ex.flow(&f, d, 1);
}

template<class Exec>
void
quant_weights_self(Exec& ex, const QwFlowFn& f, long)
{
  ex.foreach(1, QuantWeightSeqFn{f.preds, f.qw, f.start, f.end, f.nw});
}

// computeQuantizationWeightsScalable (PCCTMC3Common.h:858-891): one constant
// per level of detail
struct QuantWeightScalableFn {
  uint64_t* qw;
  int64_t start;
  uint64_t value;
  PCC_HD void operator()(int64_t i) const { qw[start + i] = value; }
};

struct LiftPredictFn {
  const pccb200_predictor* preds;
  int64_t* attr;
  int64_t start;
  int A;
  int direct;
  PCC_HD void operator()(int64_t i) const
  {
    const int64_t idx = start + i;
    const pccb200_predictor& p = preds[idx];
    for (int k = 0; k < A; k++) {
      int64_t acc = 0;
      for (uint32_t j = 0; j < p.neighbor_count; j++)
        acc += int64_t(p.weight[j]) * attr[int64_t(p.predictor_index[j]) * A + k];
      acc = div_exp2_round_half_inf(acc, 8);
      if (direct)
        attr[idx * A + k] -= acc;
      else
        attr[idx * A + k] += acc;
    }
  }
};

struct LiftUpdateScatterFn {
  const pccb200_predictor* preds;
  const uint64_t* qw;
  const int64_t* attr;
  uint64_t* updW;  // [start]
  uint64_t* upd;   // [start * A]
  int64_t start;
  int A;
  PCC_HD void operator()(int64_t i) const
  {
    const int64_t idx = start + i;
    const pccb200_predictor& p = preds[idx];
    const uint64_t q = qw[idx];
    for (uint32_t j = 0; j < p.neighbor_count; j++) {
      const uint64_t w = div_exp2_round_half_inf_u(uint64_t(p.weight[j]) * q, 8);
      const int64_t nb = p.predictor_index[j];
      atomic_add_u64(&updW[nb], w);
      for (int k = 0; k < A; k++)
        atomic_add_u64(&upd[nb * A + k], w * uint64_t(attr[idx * A + k]));
    }
  }
};

struct LiftUpdateApplyFn {
  const uint64_t* updW;
  const uint64_t* upd;
  int64_t* attr;
  int A;
  int direct;
  PCC_HD void operator()(int64_t i) const
  {
    const uint32_t sumW = uint32_t(updW[i]);  // the reference truncates to 32 bits
    if (!sumW)
      return;
    for (int k = 0; k < A; k++) {
      int64_t u = div_approx(int64_t(upd[i * A + k]), sumW, 0);
      if (direct)
        attr[i * A + k] += u;
      else
        attr[i * A + k] -= u;
    }
  }
};

//----------------------------------------------------------------------------
// lifting quantisation + last-component prediction
//   tmc3/AttributeEncoder.cpp:1424-1473,1498-1539,1597-1625
//   tmc3/AttributeDecoder.cpp:711-749,815-837

struct LodTable {
  uint32_t npl[PCCB200_MAX_LODS];
  int lodCount;
  // level of detail of predictor i: number of cumulative sizes <= i
  PCC_HD int lod_of(int64_t i) const
  {
    int l = 0;
    while (l < lodCount && int64_t(npl[l]) <= i)
      l++;
    return l;
  }
};

// per-LoD sums for computeLastComponentPredictionCoeff (note the reference's
// truncation of the products to int)
struct LcpSumFn {
  const int64_t* coeffs;  // row i at coeffs + i * stride + off, 3 components
  int stride, off;
  LodTable lt;
  uint64_t* sums;  // [lod][2]: sum k1*k2, sum k1*k1 (two's complement)
  PCC_HD void operator()(int64_t i) const
  {
    const int64_t* c = &coeffs[i * stride + off];
    const uint64_t k1 = uint64_t(c[1]), k2 = uint64_t(c[2]);
    const int32_t m12 = int32_t(uint32_t(k1 * k2));
    const int32_t m11 = int32_t(uint32_t(k1 * k1));
    const int l = lt.lod_of(i);
#if defined(__CUDA_ARCH__)
    // a warp whose 32 coefficients belong to one level of detail (nearly all of
    // them) adds once: the sums are modulo 2^64, so the order does not matter
    if (__activemask() == 0xffffffffu && __match_any_sync(0xffffffffu, l) == 0xffffffffu) {
      long long a = m12, b = m11;
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      if ((threadIdx.x & 31) == 0) {
        atomic_add_u64(&sums[2 * l], uint64_t(a));
        atomic_add_u64(&sums[2 * l + 1], uint64_t(b));
      }
      return;
    }
#endif
    atomic_add_u64(&sums[2 * l], uint64_t(int64_t(m12)));
    atomic_add_u64(&sums[2 * l + 1], uint64_t(int64_t(m11)));
  }
};

struct LiftQuantFn {
  int forward;
  int A;
  int stride, off;  // coefficient row i at attrs + i * stride + off
  LayerQp layers[PCCB200_MAX_QP_LAYERS];
  int numLayers;
  LodTable lt;
  int lcp[PCCB200_MAX_LODS + 1];
  const int32_t* qpo;      // n*2 in predictor order, or null
  const uint64_t* qw;
  int64_t* attrs;          // coefficients in / reconstructed coefficients out
  int32_t* values;         // n*A quantised values (out when forward, in otherwise)
  PCC_HD void operator()(int64_t i) const
  {
    const int l = lt.lod_of(i);
    const int layer = l < numLayers - 1 ? l : numLayers - 1;
    Quantizer q[2];
    make_quantizers(layers[layer], qpo ? qpo[2 * i] : 0, qpo ? qpo[2 * i + 1] : 0, q);
    const int64_t iqw = int64_t(irsqrt64(qw[i]));
    const int64_t qwt = int64_t((qw[i] * uint64_t(iqw) + (uint64_t(1) << 39)) >> 40);
    int64_t* a = &attrs[i * stride + off];
    int32_t* v = &values[i * A];
    if (forward)
      v[0] = int32_t(q[0].quantize(a[0] * qwt));
    a[0] = div_exp2_round_half_inf(q[0].scale(v[0]) * iqw, 40);
    if (A == 1)
      return;
    const int64_t c = lcp[l];
    if (forward)
      v[1] = int32_t(q[1].quantize(a[1] * qwt));
    int64_t scaled = q[1].scale(v[1]);
    a[1] = div_exp2_round_half_inf(scaled * iqw, 40);
    if (forward)
      a[2] -= (c * a[1]) >> 2;
    scaled = (scaled * c) >> 2;
    if (forward)
      v[2] = int32_t(q[1].quantize(a[2] * qwt));
    scaled += q[1].scale(v[2]);
    a[2] = div_exp2_round_half_inf(scaled * iqw, 40);
  }
};

// computeLastComponentPredictionCoeff from the per-LoD sums (host, tiny)
inline void
lcp_from_sums(const int64_t* sums, int lodCount, int numDetailLevels, int8_t* out)
{
  int lod = 0;
  for (; lod < lodCount && lod < numDetailLevels; lod++) {
    const int64_t s12 = sums[2 * lod], s11 = sums[2 * lod + 1];
    int scale = 0;
    if (s12 && s11) {
      const int sign = ((s12 < 0) ^ (s11 < 0)) ? -1 : 1;
      scale = int(((s12 << 2) + sign * (s11 >> 1)) / s11);
    }
    out[lod] = int8_t(scale < -8 ? -8 : (scale > 8 ? 8 : scale));
  }
  for (; lod < numDetailLevels; lod++)
    out[lod] = lod ? out[lod - 1] : 0;
}

// attrs: A coefficients per point at attrs + i * stride + off (executor
// memory; stride = A, off = 0 for one attribute, or one attribute's columns of
// rows holding several).  lcpInOut: host array of numDetailLevels entries;
// computed when forward && lcpEnabled, read when !forward && lcpEnabled.
template<class Exec>
int
run_lift_quant(Exec& ex, bool forward, const pccb200_qpset& qs, const int32_t* qpo,
               const uint64_t* qw, int64_t n, const uint32_t* numPointsInLod, int lodCount,
               int numDetailLevels, int64_t* attrs, int stride, int off, int A, bool lcpEnabled,
               int8_t* lcpInOut, int32_t* values)
{
  if (lodCount < 1 || lodCount > PCCB200_MAX_LODS || numDetailLevels < lodCount
      || numDetailLevels > PCCB200_MAX_LODS || qs.num_layers < 1
      || qs.num_layers > PCCB200_MAX_QP_LAYERS || (A != 1 && A != 3) || off < 0
      || off + A > stride)
    return PCCB200_ERR_INVALID_ARG;
  ex.phase(5);
  LiftQuantFn fn;
  fn.forward = forward;
  fn.A = A;
  fn.stride = stride;
  fn.off = off;
  fn.numLayers = qs.num_layers;
  for (int i = 0; i < qs.num_layers; i++) {
    fn.layers[i].luma = qs.layers[i][0];
    fn.layers[i].chromaOffset = qs.layers[i][1];
    fn.layers[i].maxQp = qs.max_qp;
    fn.layers[i].fixedPointQpOffset = qs.fixed_point_qp_offset;
  }
  // The reference advances its per-LoD counters with `if (i == npl[lod]) lod++`
  // (tmc3/AttributeEncoder.cpp:1429-1437,1514-1515): an empty level of detail
  // (two equal cumulative sizes) is never stepped over, so only the strictly
  // increasing prefix of the table takes effect.
  int effCount = 0;
  while (effCount < lodCount
         && numPointsInLod[effCount] > (effCount ? numPointsInLod[effCount - 1] : 0u))
    effCount++;
  fn.lt.lodCount = effCount;
  for (int l = 0; l < effCount; l++)
    fn.lt.npl[l] = numPointsInLod[l];
  for (int l = 0; l <= PCCB200_MAX_LODS; l++)
    fn.lcp[l] = 0;
  if (lcpEnabled && A == 3) {
    if (forward) {
      uint64_t* dSums = ex.template alloc<uint64_t>(2 * PCCB200_MAX_LODS + 2);
      ex.zero(dSums, (2 * PCCB200_MAX_LODS + 2) * sizeof(uint64_t));
      ex.foreach(n, LcpSumFn{attrs, stride, off, fn.lt, dSums});
      int64_t sums[2 * PCCB200_MAX_LODS + 2];
      ex.download(sums, dSums, sizeof(sums));
      lcp_from_sums(sums, effCount, numDetailLevels, lcpInOut);
    }
    for (int l = 0; l < numDetailLevels; l++)
      fn.lcp[l] = lcpInOut[l];
    fn.lcp[numDetailLevels] = lcpInOut[numDetailLevels - 1];
  }
  fn.qpo = qpo;
  fn.qw = qw;
  fn.attrs = attrs;
  fn.values = values;
  ex.foreach(n, fn);
  return PCCB200_OK;
}

// predictor order <-> point order helpers of the attribute-level calls.  The
// coefficient rows (stride components per point) may hold several attributes:
// one attribute's A components start at column off.
struct GatherAttrShiftFn {   // out[i][off + k] = in[indexes[i]][k] << 8
  const int32_t* in;
  const uint32_t* indexes;
  int A;
  int stride, off;
  int64_t* out;
  PCC_HD void operator()(int64_t i) const
  {
    for (int k = 0; k < A; k++)
      out[i * stride + off + k] = int64_t(in[size_t(indexes[i]) * A + k]) << 8;
  }
};
struct GatherQpoFn {
  const int32_t* in;
  const uint32_t* indexes;
  int32_t* out;
  PCC_HD void operator()(int64_t i) const
  {
    out[2 * i] = in[2 * size_t(indexes[i])];
    out[2 * i + 1] = in[2 * size_t(indexes[i]) + 1];
  }
};
struct ScatterReconFn {  // out[indexes[i]][k] = clip(divExp2RoundHalfInf(in[i][off + k], 8))
  const int64_t* in;
  const uint32_t* indexes;
  int A;
  int stride, off;
  int32_t clipMax;
  int32_t* out;
  PCC_HD void operator()(int64_t i) const
  {
    for (int k = 0; k < A; k++) {
      int64_t v = div_exp2_round_half_inf(in[i * stride + off + k], 8);
      v = v < 0 ? 0 : (v > clipMax ? clipMax : v);
      out[size_t(indexes[i]) * A + k] = int32_t(v);
    }
  }
};

// executor-generic drivers (numPointsInLod is a host array)

template<class Exec>
int
run_quant_weights(Exec& ex, const pccb200_predictor* preds, int64_t n,
                  const uint32_t* numPointsInLod, int lodCount, uint64_t* qw,
                  const int32_t* fixedNeighWeight = nullptr)
{
  NeighWeights nw{{0, 0, 0}, 0};
  if (fixedNeighWeight) {
    for (int j = 0; j < 3; j++)
      nw.fixed[j] = fixedNeighWeight[j];
    nw.useFixed = 1;
  }
  ex.phase(5);
  ex.foreach(n, FillU64Fn{qw, uint64_t(1) << 8});
  int* dFlags = ex.template alloc<int>(size_t(lodCount) + 1);
  ex.zero(dFlags, (size_t(lodCount) + 1) * sizeof(int));
  int64_t prevEnd = 0;
  for (int l = 0; l < lodCount; l++) {
    int64_t s = l ? numPointsInLod[l - 1] : 0;
    int64_t e = numPointsInLod[l];
    if (s != prevEnd || e < s || e > n)
      return PCCB200_ERR_INVALID_ARG;
    prevEnd = e;
    ex.foreach(e - s, LodCheckFn{preds, s, dFlags + l, n});
  }
  if (prevEnd != n)
    return PCCB200_ERR_INVALID_ARG;
  std::vector<int> flags(size_t(lodCount) + 1);
  ex.download(flags.data(), dFlags, flags.size() * sizeof(int));
  for (int l = 0; l < lodCount; l++)
    if (flags[l] & 2)
      return PCCB200_ERR_INVALID_ARG;
  int* cnt = nullptr;
  for (int l = lodCount - 1; l >= 0; l--) {
    int64_t s = l ? numPointsInLod[l - 1] : 0;
    int64_t e = numPointsInLod[l];
    // (a reference to a higher index has no dataflow order: one ordered walk)
    if (flags[l] & 4) {
      ex.foreach(1, QuantWeightSeqFn{preds, qw, s, e, nw});
    } else if (flags[l]) {
      if (!cnt)
        cnt = ex.template alloc<int>(size_t(n));
      quant_weights_self(ex, QwFlowFn{preds, qw, cnt, s, e, nw, nullptr}, 0);
    } else
      ex.foreach(e - s, QuantWeightLodFn{preds, qw, s, nw});
  }
  return PCCB200_OK;
}

// PCCB200_ERR_INVALID_ARG unless indexes[n] is a permutation of [0, n) and
// every predictor has at most three neighbours, all of them in [0, n)
template<class Exec>
int
run_lod_import_check(Exec& ex, const pccb200_predictor* preds, const uint32_t* indexes, int64_t n)
{
  int* seen = ex.template alloc<int>(size_t(n) + 1);
  ex.zero(seen, (size_t(n) + 1) * sizeof(int));
  int* dFlag = seen + n;
  ex.foreach(n, LodImportCheckFn{preds, indexes, seen, dFlag, n});
  int flag = 0;
  ex.download(&flag, dFlag, sizeof(int));
  return flag ? PCCB200_ERR_INVALID_ARG : PCCB200_OK;
}

template<class Exec>
int
run_quant_weights_scalable(Exec& ex, const uint32_t* numPointsInLod, int lodCount,
                           uint64_t numPoints, int minGeomNodeSizeLog2, int64_t n, uint64_t* qw)
{
  ex.phase(5);
  int64_t prevEnd = 0;
  for (int l = 0; l < lodCount; l++) {
    const int64_t s = l ? numPointsInLod[l - 1] : 0;
    const int64_t e = numPointsInLod[l];
    if (s != prevEnd || e < s || e > n || e == 0)
      return PCCB200_ERR_INVALID_ARG;
    prevEnd = e;
    uint64_t v = (numPoints / uint64_t(e)) << 8;
    if (!minGeomNodeSizeLog2 && l == lodCount - 1)
      v = uint64_t(1) << 8;
    ex.foreach(e - s, QuantWeightScalableFn{qw, s, v});
  }
  return prevEnd == n ? PCCB200_OK : PCCB200_ERR_INVALID_ARG;
}

// attr: n rows of A coefficients, predictor order.  Every component goes
// through the same arithmetic, and the update weights depend on the predictors
// and the quantisation weights only, so a row may hold several attributes side
// by side (A = their total component count): each attribute comes out
// bit-identical to a pass of its own, for the launches of one pass.
template<class Exec>
int
run_lift(Exec& ex, bool forward, const pccb200_predictor* preds, const uint64_t* qw,
         int64_t n, const uint32_t* numPointsInLod, int lodCount, int64_t* attr, int A)
{
  if (lodCount < 1 || int64_t(numPointsInLod[lodCount - 1]) != n)
    return PCCB200_ERR_INVALID_ARG;
  ex.phase(5);
  // the lifting passes require strictly-coarser references
  int* dFlag = ex.template alloc<int>(1);
  ex.zero(dFlag, sizeof(int));
  for (int l = 1; l < lodCount; l++) {
    int64_t s = numPointsInLod[l - 1], e = numPointsInLod[l];
    if (e < s || e > n)
      return PCCB200_ERR_INVALID_ARG;
    ex.foreach(e - s, LodCheckFn{preds, s, dFlag, n});
  }
  int flag = 0;
  ex.download(&flag, dFlag, sizeof(int));
  if (flag & 2)
    return PCCB200_ERR_INVALID_ARG;
  if (flag)
    return PCCB200_ERR_UNSUPPORTED;

  int64_t maxStart = lodCount > 1 ? numPointsInLod[lodCount - 2] : 0;
  uint64_t* updW = ex.template alloc<uint64_t>(size_t(maxStart));
  uint64_t* upd = ex.template alloc<uint64_t>(size_t(maxStart) * A);
  auto update = [&](int64_t s, int64_t e, bool direct) {
    ex.zero(updW, size_t(s) * sizeof(uint64_t));
    ex.zero(upd, size_t(s) * A * sizeof(uint64_t));
    ex.foreach(e - s, LiftUpdateScatterFn{preds, qw, attr, updW, upd, s, A});
    ex.foreach(s, LiftUpdateApplyFn{updW, upd, attr, A, direct});
  };
  if (forward) {
    for (int l = lodCount - 1; l >= 1; l--) {
      int64_t s = numPointsInLod[l - 1], e = numPointsInLod[l];
      ex.foreach(e - s, LiftPredictFn{preds, attr, s, A, 1});
      update(s, e, true);
    }
  } else {
    for (int l = 1; l < lodCount; l++) {
      int64_t s = numPointsInLod[l - 1], e = numPointsInLod[l];
      update(s, e, false);
      ex.foreach(e - s, LiftPredictFn{preds, attr, s, A, 0});
    }
  }
  return PCCB200_OK;
}

}  // namespace pccb200
