/* pred_oracle.c — TEST INFRASTRUCTURE ONLY (oracle).
 *
 * Sequential plain-C restatement of the predicting transform's decoder after
 * its entropy decoding, point by point in coding order:
 *   decodeReflectancesPred        tmc3/AttributeDecoder.cpp:328-391
 *   decodeColorsPred              tmc3/AttributeDecoder.cpp:446-523
 *   decodePredModeRefl / Color    tmc3/AttributeDecoder.cpp:289-323,396-441
 *   predModeEligibleColor / Refl  tmc3/AttributeCommon.cpp:145-210
 *   predictColor / Reflectance    tmc3/PCCTMC3Common.h:526-587
 *   computeQuantizationWeights    tmc3/PCCTMC3Common.h:895-921
 *   adaptivePredictionThreshold   tmc3/hls.h:808-811
 *   QpSet::quantizers             tmc3/quantization.cpp:165-188
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/pcc_attr_b200.h"
#include "pcc_arith_oracle.h"

void oracle_quant_weights_fixed(const pccb200_predictor* preds, int n, const int32_t neigh_weight[3],
                                uint64_t* qw);

static void
pred_quantizers(const pccb200_qpset* qs, int layer, int off0, int off1, orc_quantizer q[2])
{
  int qp0 = qs->layers[layer][0] + off0;
  qp0 = qp0 < 4 ? 4 : (qp0 > qs->max_qp ? qs->max_qp : qp0);
  int qp1 = qs->layers[layer][1] + off1 + qp0;
  qp1 = qp1 < 4 ? 4 : (qp1 > qs->max_qp ? qs->max_qp : qp1);
  q[0] = orc_mkquant(qp0 + qs->fixed_point_qp_offset);
  q[1] = orc_mkquant(qp1 + qs->fixed_point_qp_offset);
}

/* decodePredModeColor (coeff[1], coeff[2]) or decodePredModeRefl (coeff[0]) */
static int
pred_mode(const pccb200_pred_params* pp, int A, int32_t* v)
{
  const int maxcand = pp->max_num_direct_predictors + !pp->direct_avg_predictor_disabled;
  int mode = 0;
  if (A == 3) {
    const int s1 = v[1] < 0 ? -1 : 1, s2 = v[2] < 0 ? -1 : 1;
    const int a1 = abs(v[1]), a2 = abs(v[2]);
    switch (maxcand) {
    case 4:
      v[1] = s1 * (a1 >> 1);
      v[2] = s2 * (a2 >> 1);
      mode = ((a1 & 1) << 1) + (a2 & 1);
      break;
    case 3:
      v[1] = s1 * (a1 >> 1);
      mode = a1 & 1;
      if (a1 & 1) {
        v[2] = s2 * (a2 >> 1);
        mode += a2 & 1;
      }
      break;
    case 2:
      v[1] = s1 * (a1 >> 1);
      mode = a1 & 1;
      break;
    default: mode = 0;
    }
  } else {
    const int s = v[0] < 0 ? -1 : 1;
    int a = abs(v[0]);
    switch (maxcand) {
    case 4:
      mode = a & 3;
      v[0] = s * (a >> 2);
      break;
    case 3:
      mode = a & 1;
      a >>= 1;
      if (mode > 0) {
        mode += a & 1;
        a >>= 1;
      }
      v[0] = s * a;
      break;
    case 2:
      mode = a & 1;
      v[0] = s * (a >> 1);
      break;
    default: mode = 0;
    }
  }
  return mode + (pp->direct_avg_predictor_disabled ? 1 : 0);
}

/* preds / indexes / npl: the levels of detail (predictor order, lodCount
 * cumulative counts); qpo: n x 2 in point order or NULL; icp: PCCB200_MAX_LODS
 * x 3 or NULL (no icpCoeffs); values: n x A in coding order; out: n x A in
 * point order.  Returns 0. */
int
oracle_pred_decode(const pccb200_predictor* preds, const uint32_t* indexes, int n,
                   const uint32_t* npl, int lodCount, const pccb200_qpset* qs,
                   const pccb200_pred_params* pp, const int32_t qnw[3], const int32_t* qpo,
                   const int8_t* icp, const int32_t* values, int A, int bitdepth, int32_t* out)
{
  uint64_t* qw = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(n ? n : 1));
  uint16_t* attr = (uint16_t*)calloc((size_t)(n ? n : 1) * A, sizeof(uint16_t));
  oracle_quant_weights_fixed(preds, n, qnw, qw);
  const int64_t clipMax = (1ll << bitdepth) - 1;
  const int threshold = pp->adaptive_prediction_threshold << (bitdepth > 8 ? bitdepth - 8 : 0);
  int quantLayer = 0, lod = 0;
  int icpCoeff[3] = {0, 0, 0};
  if (icp)
    for (int k = 0; k < 3; k++)
      icpCoeff[k] = icp[k];
  for (int i = 0; i < n; i++) {
    if (quantLayer < lodCount && (uint32_t)i == npl[quantLayer])
      quantLayer = quantLayer + 1 < qs->num_layers ? quantLayer + 1 : qs->num_layers - 1;
    const uint32_t pointIndex = indexes[i];
    orc_quantizer q[2];
    pred_quantizers(qs, quantLayer, qpo ? qpo[2 * pointIndex] : 0, qpo ? qpo[2 * pointIndex + 1] : 0,
                    q);
    const pccb200_predictor* p = &preds[i];
    int32_t v[3] = {0, 0, 0};
    for (int k = 0; k < A; k++)
      v[k] = values[(size_t)i * A + k];

    int predMode = 0;
    if (p->neighbor_count > 1 && pp->max_num_direct_predictors) {
      int64_t maxDiff = 0;
      for (int k = 0; k < A; k++) {
        int64_t lo = 0, hi = 0;
        for (uint32_t j = 0; j < p->neighbor_count; j++) {
          const int64_t x = attr[(size_t)indexes[p->predictor_index[j]] * A + k];
          if (j == 0 || x < lo)
            lo = x;
          if (j == 0 || x > hi)
            hi = x;
        }
        if (hi - lo > maxDiff)
          maxDiff = hi - lo;
      }
      if (maxDiff >= threshold)
        predMode = pred_mode(pp, A, v);
    }

    int64_t pred[3] = {0, 0, 0};
    if ((uint32_t)predMode > p->neighbor_count) {
      /* nop */
    } else if (predMode > 0) {
      const uint32_t nb = indexes[p->predictor_index[predMode - 1]];
      for (int k = 0; k < A; k++)
        pred[k] = attr[(size_t)nb * A + k];
    } else {
      for (int k = 0; k < A; k++) {
        for (uint32_t j = 0; j < p->neighbor_count; j++) {
          const uint16_t c = attr[(size_t)indexes[p->predictor_index[j]] * A + k];
          if (A == 3)
            pred[k] += (uint32_t)(p->weight[j] * c);          /* const uint32_t w */
          else
            pred[k] += (int64_t)((uint64_t)p->weight[j] * c); /* uint64_t weight */
        }
        pred[k] = orc_div_exp2_half_inf(pred[k], 8);
        if (A == 3)
          pred[k] = (uint16_t)pred[k]; /* Vec3<attr_t> */
      }
    }

    if (A == 3 && icp && (uint32_t)i == npl[lod]) {
      ++lod;
      for (int k = 0; k < 3; k++)
        icpCoeff[k] = icp[3 * lod + k];
    }

    int64_t residual0 = 0;
    for (int k = 0; k < A; k++) {
      const orc_quantizer qk = q[k < 1 ? k : 1];
      const int64_t qStep = qk.step;
      int64_t weight = (int64_t)qw[i] < qStep ? (int64_t)qw[i] : qStep;
      weight >>= 8;
      int64_t residual = orc_div_exp2_half_up(orc_scale(qk, v[k]), 8);
      residual /= weight;
      int64_t recon = pred[k] + residual;
      if (A == 3)
        recon += (icpCoeff[k] * residual0 + 2) >> 2;
      attr[(size_t)pointIndex * A + k] =
        (uint16_t)(recon < 0 ? 0 : (recon > clipMax ? clipMax : recon));
      if (!k && pp->icp_enabled)
        residual0 = residual;
    }
  }
  for (size_t i = 0; i < (size_t)n * A; i++)
    out[i] = attr[i];
  free(qw);
  free(attr);
  return 0;
}
