// emu_recolour_multi.cpp — TEST INFRASTRUCTURE ONLY: the recolouring kernel
// bodies of the product (recolour.cuh) compiled for the host and run as loops
// (see exec_host.h), for several attribute sets on the same positions.  Built
// by tests/test_recolour_multi.py into a temporary directory.
#include "exec_host.h"
#include "recolour.cuh"

// set s: srcAttrs[s] (nSrc x A[s]), bitdepth[s], out[s] (nTgt x A[s])
extern "C" int
emu_recolour_multi(const pccb200_recolour_params* rp, int numSets, const int32_t* srcXyz, int nSrc,
                   const int32_t* const* srcAttrs, const int32_t* A, const int32_t* bitdepth,
                   double scale, const int32_t* off, const int32_t* tgtXyz, int nTgt,
                   int32_t* const* out)
{
  HostExec ex;
  pccb200::RecolourSet sets[pccb200::kRecolourMaxSets] = {};
  for (int s = 0; s < numSets && s < pccb200::kRecolourMaxSets; s++)
    sets[s] = pccb200::RecolourSet{srcAttrs[s], A[s], bitdepth[s], nullptr, out[s]};
  return pccb200::recolour_run(ex, *rp, srcXyz, nSrc, scale, off, tgtXyz, nTgt, numSets, sets);
}
