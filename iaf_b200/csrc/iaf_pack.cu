// Weight preparation for the IAF step: mask o V -> per-output-channel l2 normalise -> scale,
// written straight into the packed layouts the step kernels read.  One launch for the whole
// stack (the reference re-derives W inside the graph on every step through ~6 tiny kernels
// per conv: tf_utils/layers.py:53-60, graphy/nodes/ar.py:312-321 with 267-281).
//
// Only the 5 live taps of the 3x3 AR mask are kept (tf_utils/layers.py:134-141 ==
// graphy/nodes/ar.py:241-264): t -> (ky,kx) = (1,1) (1,2) (2,0) (2,1) (2,2); the centre tap
// carries the MADE channel mask (layers.py:115-131).  The rule itself: iaf_tap_rule (iaf_common.h).
#include "iaf_common.h"

// raw weight of canonical tap t, input channel ci (ci == cin: pad channel), output channel co; 0 where not live
__device__ __forceinline__ float iaf_masked_weight(const IafPackLayer& L, const IafVariantFlags& vf, int t, int ci, int co) {
  const IafTap tp = iaf_tap_rule(t, ci, co, L.cin, L.cout, L.zerodiag, vf.flipmask);
  return tp.live ? L.w[iaf_raw_index(vf.theano, tp.k, ci, co, L.cin, L.cout)] : 0.f;
}

__global__ void __launch_bounds__(128) iaf_pack_kernel(const __grid_constant__ IafPackParams p) {
  const IafPackLayer& L = p.layer[blockIdx.y];
  const int co = blockIdx.x;
  if (co >= L.cout) return;
  const int tid = threadIdx.x;
  const int n_real = L.cin * IAF_NTAPS;
  // pad channel: taps 1..4; flipped, also its centre, which only enters the norm (see iaf_tap_rule)
  const int n_pad = p.vf.pad_channel ? (p.vf.flipmask ? 5 : 4) : 0;
  const int t_pad0 = IAF_NTAPS - n_pad;

  // pass 1: sum of squares of the masked row
  float ss = 0.f;
  for (int e = tid; e < n_real + n_pad; e += blockDim.x) {
    float v;
    if (e < n_real) {
      const int t = e / L.cin, ci = e % L.cin;
      v = iaf_masked_weight(L, p.vf, t, ci, co);
    } else {
      v = iaf_masked_weight(L, p.vf, t_pad0 + e - n_real, L.cin, co);
    }
    ss = fmaf(v, v, ss);
  }
  __shared__ float red[128];
  red[tid] = ss;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  ss = red[0];
  float factor;
  if (!p.vf.theano)
    factor = expf(L.scale[co]) / sqrtf(fmaxf(ss, 1e-12f));        // layers.py:60, l2_normalize eps
  else
    factor = expf(3.0f * L.scale[co]) / (sqrtf(ss) + 1e-8f);      // ar.py:277-281,316 (logscale_scale = 3)

  const int col = L.head_pairs ? ((co >> 2) * 8 + L.col0 + (co & 3)) : co;
  for (int e = tid; e < n_real + n_pad; e += blockDim.x) {
    if (e < n_real) {
      const int t = e / L.cin, ci = e % L.cin;
      L.w_out[((size_t)t * L.cin + ci) * L.cout_pad + col] = iaf_masked_weight(L, p.vf, t, ci, co) * factor;
    } else {
      const int t = t_pad0 + e - n_real;
      if (t > 0) L.padw_out[(size_t)(t - 1) * L.cout_pad + col] = iaf_masked_weight(L, p.vf, t, L.cin, co) * factor;
    }
  }
  if (tid == 0) L.bias_out[col] = L.bias[co];
}

cudaError_t iaf_launch_pack(const IafPackParams& p, int max_cout, cudaStream_t stream) {
  dim3 grid(max_cout, p.n_layers);
  IAF_LAUNCH(iaf_pack_kernel, grid, 128, 0, stream, p);
  return cudaGetLastError();
}
