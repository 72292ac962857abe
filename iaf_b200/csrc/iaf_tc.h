// Tensor-core (wgmma, sm_90a) path of the IAF step: internal interface used by iaf_capi.cu.
#pragma once
#include "iaf_common.h"

struct IafTcPlan;

struct IafTcArgs {
  int mode;  // IAF_MODE_MULTICONV | IAF_MODE_STEP | IAF_MODE_LAYER | IAF_MODE_LOGP
  const float* z;  // layer mode: eps
  const float* ctx;
  const float* post_mean;
  const float* post_logsd;
  const float* prior_mean;
  const float* prior_logsd;
  float* z_out;
  float* elem_out;       // arw_logsd | kl, nullable
  float* bc_out;         // [B,C], nullable
  float* persample_out;  // [B], nullable
  float* logps_out;      // logp mode: per-element log-density, nullable (z_out / elem_out: z' / arw_logsd, nullable)
  float* hid_out[IAF_MAX_HIDDEN];  // training forward: hidden activations [B][hidden[j]][HW], nullable
  int B;
};

bool iaf_tc_supported(const iaf_desc_t* d);
int iaf_tc_plan_create(IafTcPlan** out, const iaf_desc_t* d);
void iaf_tc_plan_destroy(IafTcPlan* p);
int iaf_tc_pack(IafTcPlan* p, const float* const* w, const float* const* scale, const float* const* bias,
                cudaStream_t stream);
bool iaf_tc_mode_supported(const IafTcPlan* p, int mode);
int iaf_tc_run(IafTcPlan* p, const IafTcArgs* a, cudaStream_t stream, int* n_launches);
int iaf_tc_scratch_need(const IafTcPlan* p, int B);  // IAF_SCRATCH_*: what iaf_tc_run at batch B does to the scratch

// Data gradient of the conv stack on the tensor cores (used by iaf_bwd.cu when the shapes allow it; IAF_BWD_TC=0 keeps
// the exact-fp32 SIMT kernels).  cin / ncol: per stage, the forward layer's input channels and packed output columns.
struct IafDgPlan;
int iaf_dg_plan_create(IafDgPlan** out, const iaf_desc_t* d, const int* cin, const int* ncol, int n_stages);
void iaf_dg_plan_destroy(IafDgPlan* p);int iaf_dg_begin(IafDgPlan* p, const float* g_heads, int B, cudaStream_t stream);
int iaf_dg_stage(IafDgPlan* p, int j, const float* w_packed, int in_buf, const float* hprev, float* out, int write_image,
                 int B, cudaStream_t stream);
int iaf_wg_run(IafDgPlan* p, int j, const float* x, int g_buf, float* part, int part_stride, int ng_max, int B,
               cudaStream_t stream, int* ng_used);
bool iaf_dg_step_supported(const IafDgPlan* p);
int iaf_dg_begin_step(IafDgPlan* p, const float* z_out, const float* logsd, const float* g_zout, const float* g_logsd,
                      const float* g_logdet, float* g_z, float* hb, int head_pad, int B, cudaStream_t stream,
                      const float** bias_partials);
// the same prologue for the MADE prior's density (IAF_MODE_LOGP): the upstream G = g_logps + g_logp_bc[b,c] + g_logp[b]
// (each nullable) enters as g_z' = -z' G, g_arw_logsd = -G
int iaf_dg_begin_step_logp(IafDgPlan* p, const float* z_out, const float* logsd, const float* g_logps,
                           const float* g_logp_bc, const float* g_logp, float* g_z, float* hb, int head_pad, int B,
                           cudaStream_t stream, const float** bias_partials);
