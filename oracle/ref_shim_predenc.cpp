// ref_shim_predenc.cpp — TEST INFRASTRUCTURE ONLY (oracle).
//
// Drives the reference's own predicting-transform ENCODER bodies
//   AttributeEncoder::encodeReflectancesPred  tmc3/AttributeEncoder.cpp:750-1073
//   AttributeEncoder::encodeColorsPred        tmc3/AttributeEncoder.cpp:1076-1210
// on levels of detail the reference generates (AttributeLods::generate), and
// returns the arithmetic-coded payload, the encoder's reconstruction, the
// levels of detail (flattened) and the ICP coefficients.  As
// ref_shim_liftenc.cpp, this TU #includes the reference's AttributeEncoder.cpp
// from where it lies with `protected` / `private` opened.
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

void tmc13ref_pred_fill_aps(const pccb200_lod_params* lp, const pccb200_pred_params* pp,
                            const int32_t qnw[3], AttributeParameterSet& aps);

extern "C" int
tmc13ref_pred_encode(
  const pccb200_lod_params* lp, const pccb200_qpset* qs, const pccb200_pred_params* pp,
  const int32_t* qnw, const int32_t* xyz, const int32_t* attrs, int n, int numAttrs,
  int bitdepth,
  uint8_t* buf, int bufCap,     // the payload
  int32_t* reconOut,            // n x numAttrs, point order
  pccb200_predictor* predsOut,  // n, predictor order
  uint32_t* idxOut,             // n
  uint32_t* nplOut,             // PCCB200_MAX_LODS
  int32_t* lodCountOut,
  int8_t* icpOut)               // PCCB200_MAX_LODS x 3 (zeros when absent)
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
  AttributeInterPredParams ip;
  ip.frameDistance = 1;
  ip.enableAttrInterPred = false;
  ip.attrInterIntraSliceRDO = false;

  AttributeEncoder enc;
  enc._abh = &abh;
  enc._lods.generate(aps, abh, n - 1, 0, cloud, ip);
  AttributeContexts ctxtMem;
  ctxtMem.reset();
  PCCResidualsEncoder encoder(aps, abh, ctxtMem);
  encoder.start(sps, n);
  if (numAttrs == 3)
    enc.encodeColorsPred(desc, aps, qpSet, cloud, encoder);
  else
    enc.encodeReflectancesPred(desc, aps, qpSet, cloud, encoder, ip);
  const int len = encoder.stop();
  if (len > bufCap)
    return -1;
  memcpy(buf, encoder.arithmeticEncoder.buffer(), len);

  for (int i = 0; i < n; i++) {
    if (numAttrs == 3) {
      auto c = cloud.getColor(i);
      for (int k = 0; k < 3; k++)
        reconOut[3 * i + k] = c[k];
    } else {
      reconOut[i] = cloud.getReflectance(i);
    }
  }
  const auto& L = enc._lods;
  for (int i = 0; i < n; i++) {
    const auto& pr = L.predictors[i];
    predsOut[i] = pccb200_predictor{};
    predsOut[i].neighbor_count = pr.neighborCount;
    for (uint32_t j = 0; j < pr.neighborCount; j++) {
      predsOut[i].predictor_index[j] = pr.neighbors[j].predictorIndex;
      predsOut[i].weight[j] = uint32_t(pr.neighbors[j].weight);
    }
    idxOut[i] = L.indexes[i];
  }
  if (int(L.numPointsInLod.size()) > PCCB200_MAX_LODS)
    return -2;
  *lodCountOut = int(L.numPointsInLod.size());
  for (size_t l = 0; l < L.numPointsInLod.size(); l++)
    nplOut[l] = L.numPointsInLod[l];
  memset(icpOut, 0, PCCB200_MAX_LODS * 3);
  if (abh.icpPresent(desc, aps))
    for (size_t l = 0; l < abh.icpCoeffs.size() && l < PCCB200_MAX_LODS; l++)
      for (int k = 0; k < 3; k++)
        icpOut[3 * l + k] = abh.icpCoeffs[l][k];
  return len;
}
