// emu_rdoq.cpp — TEST INFRASTRUCTURE ONLY: the RDOQ threshold search of the
// product (rdoq_code, raht_core.cuh) compiled for the host.  Built by
// tests/test_rdoq_threshold.py into a temporary directory.
#include "exec_host.h"

extern "C" void
emu_rdoq_codes(const int64_t* dist2, const int64_t* lambda, const int32_t* rateCoeff, int n,
               int32_t* codes)
{
  for (int i = 0; i < n; i++)
    codes[i] = pccb200::rdoq_code(dist2[i], lambda[i], 1.0f / float(lambda[i]), rateCoeff[i]);
}

extern "C" int emu_zero_run_rate(int tz) { return pccb200::zero_run_rate(tz); }
