// qpset_flatten.h — pcc::QpSet (tmc3/quantization.h) as the library's
// pccb200_qpset, shared by the drop-in translation units that hand a QpSet to
// libpcc_attr_b200.so (raht_dropin.cpp, lift_dropin.cpp).  It includes the
// reference's header; it declares nothing of its own.
#pragma once

#include <stdexcept>

#include "quantization.h"

#include "pcc_attr_b200.h"

namespace pcc {

// whether a pccb200_qpset holds qs: at least one qp layer, at most
// PCCB200_MAX_QP_LAYERS of them and PCCB200_MAX_AC_QP_LAYERS RAHT AC
// coefficient layers.  The region list is not part of a pccb200_qpset: callers
// pass QpSet::regionQpOffset per point instead.
inline bool
qpset_fits(const QpSet& qs)
{
  return !(qs.layers.empty() || int(qs.layers.size()) > PCCB200_MAX_QP_LAYERS
           || int(qs.rahtAcCoeffQps.size()) > PCCB200_MAX_AC_QP_LAYERS);
}

// q <- qs; throws std::runtime_error when !qpset_fits(qs)
inline void
flatten_qpset(const QpSet& qs, pccb200_qpset& q)
{
  if (!qpset_fits(qs))
    throw std::runtime_error("pcc_attr_b200: unsupported number of qp layers");
  q = pccb200_qpset{};
  q.num_layers = int(qs.layers.size());
  for (int i = 0; i < q.num_layers; i++) {
    q.layers[i][0] = qs.layers[i][0];
    q.layers[i][1] = qs.layers[i][1];
  }
  q.max_qp = qs.maxQp;
  q.fixed_point_qp_offset = qs.fixedPointQpOffset;
  q.num_ac_coeff_qp_layers = int(qs.rahtAcCoeffQps.size());
  for (int l = 0; l < q.num_ac_coeff_qp_layers; l++)
    for (int c = 0; c < 7; c++) {
      q.ac_coeff_qps[l][c][0] = qs.rahtAcCoeffQps[l][c][0];
      q.ac_coeff_qps[l][c][1] = qs.rahtAcCoeffQps[l][c][1];
    }
}

}  // namespace pcc
