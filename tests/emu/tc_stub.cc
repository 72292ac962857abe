// Host-emulation build only (tests/emu): the wgmma path cannot be emulated, so the library reports it as unsupported
// and every plan takes the SIMT path.  TEST INFRASTRUCTURE ONLY.
#include "iaf_tc.h"

bool iaf_tc_supported(const iaf_desc_t*) { return false; }
int iaf_tc_plan_create(IafTcPlan**, const iaf_desc_t*) { return IAF_ERR_UNSUPPORTED; }
void iaf_tc_plan_destroy(IafTcPlan*) {}
int iaf_tc_pack(IafTcPlan*, const float* const*, const float* const*, const float* const*, cudaStream_t) { return IAF_ERR_UNSUPPORTED; }
bool iaf_tc_mode_supported(const IafTcPlan*, int) { return false; }
int iaf_tc_run(IafTcPlan*, const IafTcArgs*, cudaStream_t, int*) { return IAF_ERR_UNSUPPORTED; }
int iaf_dg_plan_create(IafDgPlan** out, const iaf_desc_t*, const int*, const int*, int) { *out = nullptr; return IAF_ERR_UNSUPPORTED; }
void iaf_dg_plan_destroy(IafDgPlan*) {}
int iaf_dg_begin(IafDgPlan*, const float*, int, cudaStream_t) { return IAF_ERR_UNSUPPORTED; }
int iaf_dg_stage(IafDgPlan*, int, const float*, int, const float*, float*, int, int, cudaStream_t) { return IAF_ERR_UNSUPPORTED; }
int iaf_wg_run(IafDgPlan*, int, const float*, int, float*, int, int, int, cudaStream_t, int*) { return IAF_ERR_UNSUPPORTED; }
bool iaf_dg_step_supported(const IafDgPlan*) { return false; }
int iaf_dg_begin_step(IafDgPlan*, const float*, const float*, const float*, const float*, const float*, float*, float*, int, int,
                      cudaStream_t, const float**) { return IAF_ERR_UNSUPPORTED; }
