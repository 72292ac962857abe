// Exact-fp32 fused IAF step, SIMT FMA path (any shape; the parity anchor).
//
// One CTA = one (sample, band of rows).  The whole masked-AR stack runs out of shared
// memory: z band -> hidden_0 -> ... -> heads -> affine update -> per-channel sums; no
// intermediate touches HBM (the reference writes and re-reads every layer's activations:
// graphy/nodes/ar.py:396-416, tf_utils/layers.py:158-166, models.py:281-285).
//
// Orientation.  The TF variant's live taps read in[y+dy, x+dx] for
// (dy,dx) = (0,0)c (0,+1) (+1,-1) (+1,0) (+1,+1)  (cross-correlation, layers.py:64).
// The Theano variant's true convolution (ar.py:323) reads the point reflection of that
// set, so it is run as the TF form on the point-reflected image: loads and stores map
// pixel p -> H*W-1-p ("flip"), nothing else changes.  Zero rows/columns around the band
// give the SAME / pad2dwithchannel zero padding; the Theano pad channel (conv.py:71-83)
// is a position-dependent bias added in the epilogue.  With flipmask (the mask reversed,
// ar.py:263-264) the true convolution reads the TF offsets themselves: no reflection, the
// pad-channel bias kept (IafVariantFlags, iaf_common.h).
//
// Dependencies only look forward (down/right), so a band of R output rows needs R+1 rows
// of the last hidden layer, R+2 of the one before, ... : halo rows are recomputed, never
// exchanged.
#include "iaf_common.h"

#define IAF_PX 8   // consecutive x per thread tile
#define IAF_CT 8   // output channels per thread tile
#define IAF_SIMT_THREADS 256

#define IAF_TAP(T, A, OFF)                                                        \
  {                                                                               \
    const float4 wa = __ldg(reinterpret_cast<const float4*>(wrow + (T) * tapstride));      \
    const float4 wb = __ldg(reinterpret_cast<const float4*>(wrow + (T) * tapstride) + 1);  \
    _Pragma("unroll") for (int j = 0; j < IAF_PX; ++j) {                          \
      const float a = A[j + OFF];                                                 \
      acc[j][0] = fmaf(a, wa.x, acc[j][0]); acc[j][1] = fmaf(a, wa.y, acc[j][1]); \
      acc[j][2] = fmaf(a, wa.z, acc[j][2]); acc[j][3] = fmaf(a, wa.w, acc[j][3]); \
      acc[j][4] = fmaf(a, wb.x, acc[j][4]); acc[j][5] = fmaf(a, wb.y, acc[j][5]); \
      acc[j][6] = fmaf(a, wb.z, acc[j][6]); acc[j][7] = fmaf(a, wb.w, acc[j][7]); \
    }                                                                             \
  }

// LOGP: the MADE prior's density (IAF_MODE_LOGP), an instantiation of its own so that the other modes' code is untouched
template <bool LOGP>
__global__ void __launch_bounds__(IAF_SIMT_THREADS, 2) iaf_simt_kernel(const __grid_constant__ IafSimtParams p) {
  IAF_DYN_SMEM(float, smem);
  float* bufz = smem;
  float* bufa = bufz + p.bufz_elems;
  float* bufb = bufa + p.bufa_elems;
  float* tilepart = bufb + p.bufb_elems;  // [ntiles_last][4]
  __shared__ float s_chan[256];
  __shared__ unsigned s_last;

  const int tid = threadIdx.x;
  const int n = blockIdx.x / p.n_bands, band = blockIdx.x % p.n_bands;
  const int H = p.H, W = p.W, HW = H * W, P = p.P, C = p.C;
  const int r0 = band * p.band_rows;
  const int R = min(p.band_rows, H - r0);
  const int nst = p.n_stages;
  const int rows_alloc = p.band_rows + nst;  // rows per channel plane in every smem buffer
  const int nseg = (W + IAF_PX - 1) / IAF_PX;

  // ---- stage in the z band (rows r0 .. r0+R+nst-1, clipped; everything else stays 0) ----
  for (int i = tid; i < p.bufz_elems; i += IAF_SIMT_THREADS) bufz[i] = 0.f;
  __syncthreads();
  {
    const int nrows = min(H - r0, R + nst);
    const int total = C * nrows * W;
    for (int i = tid; i < total; i += IAF_SIMT_THREADS) {
      const int x = i % W;
      const int l = (i / W) % nrows;
      const int c = i / (W * nrows);
      const int pix = (r0 + l) * W + x;
      const size_t g = ((size_t)n * C + c) * HW + (p.flip ? HW - 1 - pix : pix);
      float v = __ldg(p.z + g);
      if (p.mode == IAF_MODE_LAYER)  // z0 = mean + exp(.5*logvar)*eps, logvar = 2*logsd  (tf_train.py:57, distributions.py:20)
        v = fmaf(expf(__ldg(p.post_logsd + g)), v, __ldg(p.post_mean + g));
      bufz[(c * rows_alloc + l) * P + x + 1] = v;
    }
  }
  __syncthreads();

  const float* in = bufz;
  for (int js = 0; js < nst; ++js) {
    const IafStageDev& S = p.stage[js];
    const bool last = (js == nst - 1);
    const int ro = min(H - r0, R + (nst - 1 - js));  // output rows of this stage
    float* out = (js & 1) ? bufb : bufa;
    if (!last) {
      const int nz = S.cout * rows_alloc * P;
      for (int i = tid; i < nz; i += IAF_SIMT_THREADS) out[i] = 0.f;
      __syncthreads();
    }
    const int nct = S.cout_pad / IAF_CT;
    const int ntiles = ro * nseg * nct;
    const size_t tapstride = (size_t)S.cin * S.cout_pad;
    const int plane = rows_alloc * P;

    for (int tile = tid; tile < ntiles; tile += IAF_SIMT_THREADS) {
      const int ct = tile % nct;
      const int t2 = tile / nct;
      const int seg = t2 % nseg;
      const int yl = t2 / nseg;
      float acc[IAF_PX][IAF_CT];
#pragma unroll
      for (int j = 0; j < IAF_PX; ++j)
#pragma unroll
        for (int c = 0; c < IAF_CT; ++c) acc[j][c] = 0.f;

      const float* a0p = in + yl * P + seg * IAF_PX + 1;    // row y   : cols x0 .. x0+8
      const float* a1p = in + (yl + 1) * P + seg * IAF_PX;  // row y+1 : cols x0-1 .. x0+8
      const float* wrow = S.w + ct * IAF_CT;
      for (int ci = 0; ci < S.cin; ++ci) {
        float a0[IAF_PX + 1], a1[IAF_PX + 2];
#pragma unroll
        for (int j = 0; j < IAF_PX + 1; ++j) a0[j] = a0p[j];
#pragma unroll
        for (int j = 0; j < IAF_PX + 2; ++j) a1[j] = a1p[j];
        IAF_TAP(0, a0, 0)  // ( 0, 0) centre, MADE-masked
        IAF_TAP(1, a0, 1)  // ( 0,+1)
        IAF_TAP(2, a1, 0)  // (+1,-1)
        IAF_TAP(3, a1, 1)  // (+1, 0)
        IAF_TAP(4, a1, 2)  // (+1,+1)
        a0p += plane;
        a1p += plane;
        wrow += S.cout_pad;
      }

      // ---- epilogue ----
      const int y = r0 + yl;
      const bool byH = (y == H - 1);
      if (!last) {
#pragma unroll
        for (int j = 0; j < IAF_PX; ++j) {
          const int x = seg * IAF_PX + j;
          if (x >= W) continue;
          const bool bx0 = (x == 0), bxW = (x == W - 1);
          const int pix = y * W + x;
          const int gp = p.flip ? HW - 1 - pix : pix;
#pragma unroll
          for (int c = 0; c < IAF_CT; ++c) {
            const int co = ct * IAF_CT + c;
            if (co >= S.cout) continue;
            float v = acc[j][c] + __ldg(S.bias + co);
            if (S.padw) {  // pad channel = 1 where the tap falls outside the image (conv.py:77-83)
              if (bxW) v += __ldg(S.padw + co);
              if (byH || bx0) v += __ldg(S.padw + S.cout_pad + co);
              if (byH) v += __ldg(S.padw + 2 * S.cout_pad + co);
              if (byH || bxW) v += __ldg(S.padw + 3 * S.cout_pad + co);
            }
            if (js == 0) v += __ldg(p.ctx + ((size_t)n * S.cout + co) * HW + gp);  // ar.py:402 / layers.py:163
            v = iaf_apply_nl(v, p.nl);
            out[(co * rows_alloc + yl) * P + x + 1] = v;
            // training forward: keep the activations (rows of this band only; halo rows belong to the next band)
            if (p.hid_out[js] && yl < R) p.hid_out[js][((size_t)n * S.cout + co) * HW + gp] = v;
          }
        }
      } else {
        float csum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < IAF_PX; ++j) {
          const int x = seg * IAF_PX + j;
          if (x >= W) continue;
          const bool bx0 = (x == 0), bxW = (x == W - 1);
          const int pix = y * W + x;
          const int gp = p.flip ? HW - 1 - pix : pix;
          float o[IAF_CT];
#pragma unroll
          for (int c = 0; c < IAF_CT; ++c) {
            const int col = ct * IAF_CT + c;
            float v = acc[j][c] + __ldg(S.bias + col);
            if (S.padw) {
              if (bxW) v += __ldg(S.padw + col);
              if (byH || bx0) v += __ldg(S.padw + S.cout_pad + col);
              if (byH) v += __ldg(S.padw + 2 * S.cout_pad + col);
              if (byH || bxW) v += __ldg(S.padw + 3 * S.cout_pad + col);
            }
            o[c] = v;
          }
          if (p.n_heads == 1) {
            if (p.mode == IAF_MODE_MULTICONV) {
#pragma unroll
              for (int c = 0; c < IAF_CT; ++c) {
                const int ch = ct * IAF_CT + c;
                if (ch < p.head_c) p.m_out[((size_t)n * p.head_c + ch) * HW + gp] = o[c];
              }
            }
            continue;
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int ch = ct * 4 + c;
            if (ch >= p.head_c) continue;
            const size_t g = ((size_t)n * p.head_c + ch) * HW + gp;
            if (p.mode == IAF_MODE_MULTICONV) {
              p.m_out[g] = o[c];
              p.s_out[g] = o[4 + c];
              continue;
            }
            // models.py:282-285 / tf_train.py:70-72
            const float arw_mean = p.scale * o[c];
            const float arw_logsd = p.scale * o[4 + c];
            const float zv = bufz[(ch * rows_alloc + yl) * P + x + 1];
            const float zn = (zv - arw_mean) / expf(arw_logsd);
            if (!LOGP || p.z_out) p.z_out[g] = zn;
            if (LOGP) {
              // models.py:304-309, rand.py:83: N(0.1 m, exp(2 arw_logsd)) at z is the standard normal at z', - arw_logsd
              const float lp = -0.9189385332046727f - arw_logsd - 0.5f * zn * zn;
              if (p.logsd_out) p.logsd_out[g] = arw_logsd;
              if (p.logps_out) p.logps_out[g] = lp;
              csum[c] += lp;
            } else if (p.mode == IAF_MODE_STEP) {
              if (p.logsd_out) p.logsd_out[g] = arw_logsd;
              csum[c] += arw_logsd;
            } else {
              // logqs of the pre-flow sample (distributions.py:10 with (z0-mean)/sd == eps), + arw_logsd;
              // prior logps at z' (tf_train.py:68-75, models.py:277-298,328)
              const float e = __ldg(p.z + g);
              const float logqs = -0.9189385332046727f - __ldg(p.post_logsd + g) - 0.5f * e * e + arw_logsd;
              const float pl = __ldg(p.prior_logsd + g);
              const float d = zn - __ldg(p.prior_mean + g);
              const float logps = -0.9189385332046727f - pl - 0.5f * d * d * expf(-2.0f * pl);
              const float kl = logqs - logps;
              if (p.logsd_out) p.logsd_out[g] = kl;
              csum[c] += kl;
            }
          }
        }
        if (p.mode != IAF_MODE_MULTICONV && p.n_heads == 2) {
#pragma unroll
          for (int c = 0; c < 4; ++c) tilepart[tile * 4 + c] = csum[c];
        }
      }
    }
    __syncthreads();
    in = out;
  }

  if (p.mode == IAF_MODE_MULTICONV) return;

  // ---- deterministic reductions: per-channel over this band, then over bands ----
  {
    const int nct = p.stage[nst - 1].cout_pad / IAF_CT;
    if (tid < p.head_c) {
      float s = 0.f;
      const int ct = tid >> 2, c = tid & 3;
      for (int t2 = 0; t2 < R * nseg; ++t2) s += tilepart[(t2 * nct + ct) * 4 + c];
      s_chan[tid] = s;
    }
    __syncthreads();
    // logdet = -sum(arw_logsd); kl_cost = +sum(kl); logp = +sum(logps)
    const float sign = (p.mode == IAF_MODE_STEP) ? -1.f : 1.f;
    if (p.n_bands == 1) {
      if (p.bc_out && tid < p.head_c) p.bc_out[(size_t)n * p.head_c + tid] = s_chan[tid];
      if (p.persample_out && tid == 0) {
        float s = 0.f;
        for (int c = 0; c < p.head_c; ++c) s += s_chan[c];
        p.persample_out[n] = sign * s;
      }
      return;
    }
    if (tid < p.head_c) p.partial[((size_t)n * p.n_bands + band) * p.head_c + tid] = s_chan[tid];
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(p.counter + n, 1u) == (unsigned)(p.n_bands - 1));
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid < p.head_c) {
      float s = 0.f;
      for (int b = 0; b < p.n_bands; ++b) s += __ldcg(p.partial + ((size_t)n * p.n_bands + b) * p.head_c + tid);
      s_chan[tid] = s;
      if (p.bc_out) p.bc_out[(size_t)n * p.head_c + tid] = s;
    }
    __syncthreads();
    if (tid == 0) {
      if (p.persample_out) {
        float s = 0.f;
        for (int c = 0; c < p.head_c; ++c) s += s_chan[c];
        p.persample_out[n] = sign * s;
      }
      p.counter[n] = 0u;  // ready for the next launch
    }
  }
}

cudaError_t iaf_simt_set_smem() {
  cudaError_t e = iaf_smem_optin(iaf_simt_kernel<false>);
  return e != cudaSuccess ? e : iaf_smem_optin(iaf_simt_kernel<true>);
}

cudaError_t iaf_launch_simt(const IafSimtParams& p, size_t smem_bytes, cudaStream_t stream) {
  if (p.mode == IAF_MODE_LOGP) IAF_LAUNCH(iaf_simt_kernel<true>, p.B * p.n_bands, IAF_SIMT_THREADS, smem_bytes, stream, p);
  else IAF_LAUNCH(iaf_simt_kernel<false>, p.B * p.n_bands, IAF_SIMT_THREADS, smem_bytes, stream, p);
  return cudaGetLastError();
}
