// ref_shim_scalable_dec.cpp — TEST INFRASTRUCTURE ONLY (oracle).
//
// The decoder half of ref_shim_scalable_enc.cpp: this TU #includes
// tmc3/AttributeDecoder.cpp from where it lies, with `protected` / `private`
// opened, to reach
//   decode{Colors,Reflectances}Lift   tmc3/AttributeDecoder.cpp:678-857
// with scalable lifting, a given minGeomNodeSizeLog2 and
// geom_num_points_minus1 (a partial decode), and the reference's
// PCCResidualsDecoder for the quantised values of a payload.
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

void tmc13ref_scalable_aps(
  const pccb200_lod_params* lp, int maxNeighRange, AttributeParameterSet& aps);

extern "C" int
tmc13ref_scalable_decode_values(
  const uint8_t* buf, int len, int n, int numAttrs, int32_t* valuesOut)
{
  AttributeBrickHeader abh{};
  SequenceParameterSet sps{};
  AttributeContexts ctxtMem;
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
  return 0;
}

// The decoder's generate and lifting body on the n points of xyz (the cloud a
// geometry decode that stopped at minGeomNodeSizeLog2 produced),
// geom_num_points_minus1 = geomNumPoints - 1.  buf / len: payload of
// tmc13ref_scalable_payload.  lcp: 21 entries (colour with lcpEnabled).
// reconOut: n x numAttrs, input order.
extern "C" void
tmc13ref_scalable_lift_decode(
  const pccb200_lod_params* lp, int maxNeighRange, int minGeomNodeSizeLog2, int geomNumPoints,
  const pccb200_qpset* qs, int lcpEnabled, const int8_t* lcp, const int32_t* xyz, int n,
  int numAttrs, int bitdepth, const uint8_t* buf, int len, int32_t* reconOut)
{
  AttributeParameterSet aps{};
  tmc13ref_scalable_aps(lp, maxNeighRange, aps);
  aps.last_component_prediction_enabled_flag = lcpEnabled != 0;
  AttributeBrickHeader abh{};
  if (lcpEnabled && numAttrs == 3)
    abh.attrLcpCoeffs.assign(lcp, lcp + aps.maxNumDetailLevels());
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
  for (int i = 0; i < n; i++)
    cloud[i] = point_t{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  AttributeInterPredParams ip;
  ip.frameDistance = 1;
  ip.enableAttrInterPred = false;
  ip.attrInterIntraSliceRDO = false;

  AttributeDecoder dec;
  dec._lods.generate(aps, abh, geomNumPoints - 1, minGeomNodeSizeLog2, cloud, ip);
  AttributeContexts ctxtMem;
  ctxtMem.reset();
  PCCResidualsDecoder decoder(abh, ctxtMem);
  decoder.start(sps, reinterpret_cast<const char*>(buf), len);
  if (numAttrs == 3)
    dec.decodeColorsLift(
      desc, aps, abh, qpSet, geomNumPoints - 1, minGeomNodeSizeLog2, decoder, cloud);
  else
    dec.decodeReflectancesLift(
      desc, aps, abh, qpSet, geomNumPoints - 1, minGeomNodeSizeLog2, decoder, cloud, ip);
  decoder.stop();
  for (int i = 0; i < n; i++) {
    if (numAttrs == 3) {
      auto c = cloud.getColor(i);
      for (int k = 0; k < 3; k++)
        reconOut[3 * i + k] = c[k];
    } else {
      reconOut[i] = cloud.getReflectance(i);
    }
  }
}
