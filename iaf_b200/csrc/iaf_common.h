// Internal declarations shared by the CUDA translation units of libiaf_b200.so.
#pragma once
#ifdef IAF_EMU
// Host emulation of the CUDA subset the SIMT kernels use (tests/emu/cuda_emu.h): TEST INFRASTRUCTURE ONLY, it lets the
// CPU test-suite execute the kernels' index logic without a GPU.  Never compiled into libiaf_b200.so.
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
// kernel<<<grid, block, smem, stream>>>(args...) and the dynamic shared-memory window, spelled as macros so that the
// same sources also compile under the host emulation above
#define IAF_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define IAF_DYN_SMEM(type, name) extern __shared__ __align__(16) type name[]
// 4-byte asynchronous global -> shared copy (LDGSTS), zero-filled when !valid; src must be a mapped address either way
__device__ __forceinline__ void iaf_cp_async4(float* dst, const float* src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  const int n = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(n) : "memory");
}
__device__ __forceinline__ void iaf_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void iaf_cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#endif
// Raise a kernel's dynamic shared-memory limit to everything the device allows (opt-in maximum minus the kernel's static
// shared memory).  The attribute is per kernel, not per plan: setting it to one plan's size would LOWER it for plans
// created earlier with a larger footprint, so it is only ever set to the device maximum (idempotent).
template <class K>
static inline cudaError_t iaf_smem_optin(K kernel) {
#ifdef IAF_EMU
  (void)kernel;
  return cudaSuccess;
#else
  int dev = 0, optin = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e != cudaSuccess) return e;
  cudaFuncAttributes fa;
  e = cudaFuncGetAttributes(&fa, kernel);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
#endif
}
#include <stdint.h>
#include <stdlib.h>
#include "../../include/iaf_b200.h"

#define IAF_NTAPS 5          // live taps of the 3x3 AR mask: (ky,kx) = (1,1)c (1,2) (2,0) (2,1) (2,2)
#define IAF_MAX_STAGES (IAF_MAX_HIDDEN + 1)

// What a variant means to the kernels; every plan derives it once from its desc.  The kernels always apply the TF offsets
// above (the "canonical frame"), the pad-channel table at the bottom / right borders of that frame.
//   TF:               no reflection, no pad channel, TF layout and norm.
//   THEANO:           true convolution with the mask reads the point reflection of the TF offsets: the data is reflected
//                     on load / store (pixel p <-> HW-1-p), which also puts the pad channel's top / left border at the
//                     canonical bottom / right.
//   THEANO_FLIPMASK:  the mask reversed on all four axes (ar.py:263-264) reflects the taps back: true convolution with it
//                     reads the TF offsets themselves, so there is no reflection, and the pad channel sits at the bottom
//                     / right borders of the image.  Theano layout, norm and pad channel; the channel rule: iaf_tap_rule.
struct IafVariantFlags {
  int reflect;      // data point-reflected on load / store
  int pad_channel;  // the Theano pad channel (conv.py:71-83): a [4][N] table of its taps 1..4
  int theano;       // Theano raw layout [Cout][Cin+1][3][3] and norm exp(3s) / (sqrt(ss) + 1e-8) (ar.py:267-281,316)
  int flipmask;     // the reversed mask (iaf_tap_rule)
};
static inline IafVariantFlags iaf_variant_flags(int variant) {
  IafVariantFlags f;
  f.reflect = variant == IAF_VARIANT_THEANO;
  f.pad_channel = variant != IAF_VARIANT_TF;
  f.theano = variant != IAF_VARIANT_TF;
  f.flipmask = variant == IAF_VARIANT_THEANO_FLIPMASK;
  return f;
}

// The AR mask, for every layout and both mask orders: the one copy of the rule of tf_utils/layers.py:115-141 and
// graphy/nodes/ar.py:241-276.  t: canonical tap (0 = centre); ci: input channel, ci == cin the Theano pad channel; co: output
// channel; zd: zerodiagonal (heads).  Returns k = ky*3+kx of the raw parameter entry tap t multiplies, and live: the entry
// enters the normalised kernel -- the mask keeps it and, for heads, l2normalize's zero-diagonal rows (ar.py:273-276: the
// centre of rows [0, cout/cin), or row 0 when cout < cin) do not clear it.
// flipmask: the raw tap is the point reflection (2-ky, 2-kx), and the centre follows the unflipped rule of output channel
// cout-1-co and input channel cin-ci.  So channel 0 never sees the centre, and the pad channel's centre inherits channel
// 0's column: live, although it never reaches an output (the centre of the padded input is interior, i.e. 0) -- it only
// enters the norm.  Unflipped, the pad centre is masked and the zero-diagonal rows are already masked.
struct IafTap {
  int k;
  bool live;
};
__host__ __device__ __forceinline__ IafTap iaf_tap_rule(int t, int ci, int co, int cin, int cout, int zd, int flipmask) {
  const int ky = t < 2 ? 1 : 2, kx = t == 0 ? 1 : (t == 1 ? 2 : t - 2);
  IafTap r;
  r.k = flipmask ? (2 - ky) * 3 + (2 - kx) : ky * 3 + kx;
  r.live = true;
  if (t != 0) return r;
  const int c = flipmask ? cin - ci : ci, o = flipmask ? cout - 1 - co : co;
  if (cout >= cin) {
    const int k = cout / cin, i = o / k;
    r.live = (zd ? (c < i) : (c <= i)) && !(zd && co < k);
  } else {
    const int k = cin / cout;
    r.live = (zd ? (c < o * k) : (c < (o + 1) * k)) && !(zd && co == 0);
  }
  return r;
}
// canonical tap of raw kernel position k = ky*3+kx, or -1 where the mask is zero for every channel
__host__ __device__ __forceinline__ int iaf_canonical_tap(int k, int flipmask) {
  if (flipmask) k = 8 - k;
  const int ky = k / 3, kx = k % 3;
  if (ky == 1) return kx == 1 ? 0 : (kx == 2 ? 1 : -1);
  return ky == 2 ? 2 + kx : -1;
}
// index of raw entry (k, ci, co) in the reference layout: TF [3,3,cin,cout] | Theano [cout,cin+1,3,3]
__host__ __device__ __forceinline__ size_t iaf_raw_index(int theano, int k, int ci, int co, int cin, int cout) {
  return theano ? ((size_t)co * (cin + 1) + ci) * 9 + k : ((size_t)k * cin + ci) * cout + co;
}

// the hidden layers' nonlinearity (iaf_nl), as the SIMT step and the inverse apply it
__device__ __forceinline__ float iaf_apply_nl(float v, int nl) {
  switch (nl) {
    case IAF_NL_ELU: return v < 0.f ? expm1f(v) : v;                       // nodes/__init__.py:174
    case IAF_NL_SOFTPLUS: return v > 0.f ? v + log1pf(expf(-v)) : log1pf(expf(v));
    case IAF_NL_RELU: return v >= 0.f ? v : 0.f;                            // h*(h>=0)
    case IAF_NL_TANH: return tanhf(v);
    case IAF_NL_LEAKYRELU: return v < 0.f ? 0.01f * v : v;
    default: return v;
  }
}

// One conv stage as the SIMT kernel sees it (weights already masked, normalised, scaled).
struct IafStageDev {
  const float* w;     // [5][cin][cout_pad], cout contiguous (heads: see iaf_pack.cu for the column order)
  const float* bias;  // [cout_pad]
  const float* padw;  // [4][cout_pad]: Theano pad-channel weights of taps 1..4, nullptr for TF
  int cin, cout, cout_pad;
};

struct IafSimtParams {
  // inputs
  const float* z;          // [B,C,H,W]   (layer mode: eps)
  const float* ctx;        // [B,hidden0,H,W]
  const float* post_mean;  // layer mode only
  const float* post_logsd;
  const float* prior_mean;
  const float* prior_logsd;
  // outputs (nullable)
  float* z_out;
  float* logsd_out;        // step mode: arw_logsd; layer mode: kl per element
  float* m_out;            // multiconv mode: head 0
  float* s_out;            // multiconv mode: head 1
  float* bc_out;           // layer mode: [B,C] sum over (h,w) of kl; logp mode: of logps
  float* persample_out;    // step: logdet [B]; layer: kl_cost [B]; logp: logp [B]
  float* logps_out;        // logp mode: per-element log-density (z_out / logsd_out: z' / arw_logsd, training only)
  float* hid_out[IAF_MAX_HIDDEN];  // training forward: hidden activations [B][hidden[j]][HW], nullable
  float* partial;          // [B][n_bands][C] per-band per-channel partial sums
  unsigned* counter;       // [B] band arrival counters (self-resetting)
  IafStageDev stage[IAF_MAX_STAGES];
  int n_stages;            // n_hidden + 1 (last = heads)
  int n_heads, head_c, head_pad;
  int B, C, H, W, P;       // P = smem row pitch = 8*ceil(W/8) + 2
  int band_rows, n_bands;
  int flip;                // 1: data point-reflected on load/store (IafVariantFlags::reflect)
  int nl;
  int mode;                // 0 multiconv, 1 step, 2 layer, 3 logp
  float scale;             // 0.1
  int bufz_elems, bufa_elems, bufb_elems;
};

// IAF_MODE_LOGP: the autoregressive (MADE) prior's log-density at z (models.py:304-309): the step's heads and affine
// update, then logps = -0.5 log 2pi - arw_logsd - 0.5 z'^2 (rand.py:83 with mean 0.1 m, logvar 2 arw_logsd), summed per
// (sample, channel) and per sample like the layer mode's kl.
enum { IAF_MODE_MULTICONV = 0, IAF_MODE_STEP = 1, IAF_MODE_LAYER = 2, IAF_MODE_LOGP = 3 };

// What a call at batch B would do to a set of scratch buffers sized for have_B samples (0: none yet): nothing, a first
// allocation, or a re-allocation that frees the old buffers.  Sets combine with std::max.
enum { IAF_SCRATCH_FITS = 0, IAF_SCRATCH_ALLOC = 1, IAF_SCRATCH_REALLOC = 2 };
static inline int iaf_scratch_need(int have_B, int B) {
  return B <= have_B ? IAF_SCRATCH_FITS : (have_B > 0 ? IAF_SCRATCH_REALLOC : IAF_SCRATCH_ALLOC);
}

// The SM count a plan sizes its persistent grids and split-K groups for: the device's, or min(n, it) when IAF_NUM_SMS=n
// (a whole number >= 1; any other value is ignored) is in the environment when the plan is created.  Development: with a
// small n a small batch runs many tiles per CTA, the regime of the full-size workloads.
static inline int iaf_plan_num_sms(int device_sms) {
  const char* e = getenv("IAF_NUM_SMS");
  if (!e || !*e) return device_sms;
  char* end = nullptr;
  const long n = strtol(e, &end, 10);
  if (*end != '\0' || n < 1) return device_sms;
  return n < device_sms ? (int)n : device_sms;
}

// Raw-parameter description handed to the pack kernel.
struct IafPackLayer {
  const float* w;      // reference layout (TF [3,3,Cin,Cout] | Theano [Cout,Cin+1,3,3])
  const float* scale;  // g | s
  const float* bias;   // b
  float* w_out;        // simt packed
  float* bias_out;
  float* padw_out;     // Theano only
  int cin, cout, cout_pad;
  int zerodiag;        // heads: 1
  int head_pairs;      // 1: two equal heads interleaved in groups of 4 columns (m0..3,s0..3,...)
  int head_c, head_pad;
  int col0;            // first packed column this (head) layer owns when head_pairs (0 or 4)
};

struct IafPackParams {
  IafPackLayer layer[IAF_MAX_HIDDEN + IAF_MAX_HEADS];
  int n_layers;
  IafVariantFlags vf;
};

// The inverse of the step (iaf_inv.cu): one CTA per sample walks the canonical frame in reverse raster order and, within
// a pixel, the z channels in the mask's order.  Shared memory: per stage, a two-row ring of its input [cin][2][W+2]
// (columns -1 and W and the row below the map stay zero), the stage's accumulators [cout_pad], and the per-channel
// sums of arw_logsd [C].
struct IafInvParams {
  const float* u;          // [B,C,H,W]
  const float* ctx;        // [B,hidden0,H,W]
  float* z_out;
  float* logsd_out;        // nullable
  float* logdet_out;       // nullable
  // per hidden stage j: grp[grp_off[j] + g], g = 0..C+1, is where the units of stage j that become final after z
  // channel step g-1 start (step -1: before any channel), and grp[grp_off[j] + C + 2 + i] lists the units in that order
  const int* grp;
  int grp_off[IAF_MAX_HIDDEN];
  IafStageDev stage[IAF_MAX_STAGES];
  int ring_off[IAF_MAX_STAGES], acc_off[IAF_MAX_STAGES], lds_off, smem_floats;
  int n_stages, n_units;   // n_units = sum of cout_pad
  int C, H, W;
  int flip;                // IafVariantFlags::reflect
  int descending;          // the channel order: C-1 .. 0 (flipmask) or 0 .. C-1
  int nl;
  float scale;             // 0.1
};

// The adjoint of the inverse (iaf_inv_adj_kernel, iaf_inv.cu): g_u = J^-T (g_z + A_z^T (g_logsd - g_logdet)) at
// z = inverse(u), J = d step / d z, A_z = d arw_logsd / d z.  One CTA per sample walks the canonical frame in raster
// order and, within a pixel, the z channels in the reverse of the mask's order.  Shared memory: per stage, a two-row
// ring of its output gradients [cout][2][W+2] (the heads' as [2 n_z], m and s of channel c at 2c and 2c+1; columns -1
// and W and the row above the map stay zero), then per stage the gradient accumulators of its input [cin].
struct IafInvAdjParams {
  const float* u;          // [B,C,H,W]
  const float* logsd;      // [B,C,H,W]: arw_logsd at z (the inverse's own)
  const float* hid[IAF_MAX_HIDDEN];  // hidden activations at z [B][hidden[j]][H][W] (iaf_step_fwd_train)
  const float* g_z;        // [B,C,H,W]
  const float* g_logsd;    // nullable
  const float* g_logdet;   // nullable, [B]
  float* g_u;
  // per hidden stage j: grp[grp_off[j] + k], k = 0..C+1, is where the units of stage j whose gradient is final after
  // z channel step k start (step C: before the chain), and grp[grp_off[j] + C + 2 + i] lists the units in that order
  const int* grp;
  int grp_off[IAF_MAX_HIDDEN];
  IafStageDev stage[IAF_MAX_STAGES];
  int ring_off[IAF_MAX_STAGES], acc_off[IAF_MAX_STAGES], smem_floats;
  int n_stages, n_units;   // n_units = sum of cin
  int C, H, W;
  int flip;                // IafVariantFlags::reflect
  int descending;          // the mask's channel order: C-1 .. 0 (flipmask) or 0 .. C-1 (the chain walks it backwards)
  int nl;
  float scale;             // 0.1
};

cudaError_t iaf_launch_pack(const IafPackParams& p, int max_cout, cudaStream_t stream);
// The inverse's and its adjoint's launchers and shared-memory opt-in.  iaf_inv.cu fills them in when it is linked in;
// the C ABI also builds without it (tests/test_emu_kernels.py's sanitizer build), and then iaf_step_inverse and
// iaf_step_inverse_adjoint refuse with IAF_ERR_UNSUPPORTED.
struct IafInvKernel {
  cudaError_t (*launch)(const IafInvParams& p, int B, size_t smem_bytes, cudaStream_t stream);
  cudaError_t (*set_smem)();
  cudaError_t (*launch_adj)(const IafInvAdjParams& p, int B, size_t smem_bytes, cudaStream_t stream);
};
extern IafInvKernel iaf_inv;
// The fused Adamax and Eve steps' launchers (iaf_optim.cu), registered the same way: without iaf_optim.cu linked in,
// iaf_adamax_step and iaf_eve_step validate their arguments and then refuse with IAF_ERR_UNSUPPORTED.
struct IafAdamaxKernel {
  int (*launch)(int rule, const iaf_adamax_tensor_t* tensors_host, int n_tensors, float* mom1, float* mom_max,
                float* avg, double lr, double beta1, double beta2, double avg_decay, float grad_scale, void* stream,
                uint64_t* launches);
  int (*launch_eve)(const iaf_adamax_tensor_t* tensors_host, int n_tensors, float* mom1, float* mom_max, float* delta,
                    float* avg, float* lookahead, double lr, double beta1, double beta2, double beta3, float grad_scale,
                    void* stream, uint64_t* launches);
};
extern IafAdamaxKernel iaf_adamax;
// Record a failed CUDA call for iaf_last_cuda_error() and return IAF_ERR_CUDA (iaf_capi.cu).
int iaf_record_cuda_error(cudaError_t e, const char* what);
cudaError_t iaf_launch_simt(const IafSimtParams& p, size_t smem_bytes, cudaStream_t stream);
cudaError_t iaf_simt_set_smem();
