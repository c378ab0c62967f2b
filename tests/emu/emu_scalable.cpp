// emu_scalable.cpp — TEST INFRASTRUCTURE ONLY: the scalable-lifting level-of-
// detail build (lod_pipeline.cuh) and lifting coder (lift_pipeline.cuh) of the
// product compiled for the host and run as loops (see exec_host.h).  Built by
// tests/test_scalable_lifting.py into a temporary directory.
#include <algorithm>

#include "exec_host.h"
#include "lift_pipeline.cuh"

extern "C" int
emu_lod_build_scalable(const pccb200_lod_params* lod, const pccb200_lod_scalable* scal,
                       const int32_t* xyz, int n, pccb200_predictor* preds, uint32_t* indexes,
                       uint32_t* npl, int32_t* lodCount)
{
  HostExec ex;
  int cnt = 0;
  int rc = pccb200::lod_run(ex, *lod, xyz, n, preds, indexes, npl, &cnt, scal);
  *lodCount = cnt;
  return rc;
}

// one attribute set: attrs (n x A, point order; in and out when forward, out
// otherwise), values (n x A, coding order), lcp (21 entries)
extern "C" int
emu_lift_scalable(int forward, const pccb200_lod_params* lod, const pccb200_lod_scalable* scal,
                  const pccb200_qpset* qs, int lcpEnabled, const int32_t* xyz, int n,
                  int32_t* attrs, int A, int bitdepth, int32_t* values, int8_t* lcp)
{
  HostExec ex;
  int8_t lcpLocal[PCCB200_MAX_LODS + 1] = {};
  const int levels = pccb200::kScalableLevels;
  if (!forward)
    std::copy(lcp, lcp + levels, lcpLocal);
  const pccb200::LiftSet set{A, bitdepth, qs, lcpEnabled != 0, attrs, attrs, values, lcpLocal};
  int rc = pccb200::attr_lift_run(ex, forward != 0, *lod, nullptr, xyz, n, 1, &set, scal);
  if (rc == 0 && forward)
    std::copy(lcpLocal, lcpLocal + levels, lcp);
  return rc;
}
