// emu_lift_multi.cpp — TEST INFRASTRUCTURE ONLY: the lifting coder of the
// product (lift_pipeline.cuh) compiled for the host and run as loops (see
// exec_host.h), for several attribute sets on the same levels of detail.
// Built by tests/test_lift_multi.py into a temporary directory.
#include <algorithm>

#include "exec_host.h"
#include "lift_pipeline.cuh"

// set s: qs[s], lcpEnabled[s], attrs[s] (n x A[s], point order; in and out
// when forward, out otherwise), bitdepth[s], values[s] (n x A[s], coding
// order), lcp[s] (num_detail_levels entries)
extern "C" int
emu_lift_multi(int forward, const pccb200_lod_params* lod, int numSets,
               const pccb200_qpset* const* qs, const int32_t* lcpEnabled, const int32_t* xyz,
               int n, int32_t* const* attrs, const int32_t* A, const int32_t* bitdepth,
               int32_t* const* values, int8_t* const* lcp)
{
  using pccb200::kLiftMaxSets;
  HostExec ex;
  pccb200::LiftSet sets[kLiftMaxSets] = {};
  int8_t lcpLocal[kLiftMaxSets][PCCB200_MAX_LODS + 1] = {};
  const int levels = std::min(lod->num_detail_levels, PCCB200_MAX_LODS);
  for (int s = 0; s < numSets && s < kLiftMaxSets; s++) {
    if (!forward)
      std::copy(lcp[s], lcp[s] + levels, lcpLocal[s]);
    sets[s] = pccb200::LiftSet{A[s],      bitdepth[s], qs[s],     lcpEnabled[s] != 0,
                               attrs[s],  attrs[s],    values[s], lcpLocal[s]};
  }
  int rc = pccb200::attr_lift_run(ex, forward != 0, *lod, nullptr, xyz, n, numSets, sets);
  if (rc == 0 && forward)
    for (int s = 0; s < numSets; s++)
      std::copy(lcpLocal[s], lcpLocal[s] + levels, lcp[s]);
  return rc;
}
