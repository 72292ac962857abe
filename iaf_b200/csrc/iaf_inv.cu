// Inverse of the fused IAF step, exact fp32: given u, the z with (z - 0.1 m(z)) / exp(0.1 s(z)) = u.
//
// With u = eps ~ N(0,1) and the MADE prior's stack this draws a sample of the prior (models.py:36-38, 304-309); the
// reference leaves it as a TODO and uses z = eps (models.py:338-340).
//
// The forward evaluates every position at once; the inverse is a recurrence.  In the canonical frame of iaf_simt.cu the
// live taps of output (y,x) read (y,x) (the centre, channel-masked), (y,x+1) and (y+1,x-1..x+1), so the pixels are
// solved in reverse raster order and, inside a pixel, the z channels in the mask's order (ascending; descending with
// flipmask).  One CTA owns one sample:
//   1. every stage's non-centre taps read only pixels already solved: one pass over all (stage, output) pairs puts
//      bias + pad channel + context + those taps into the stage's accumulator;
//   2. for each z channel c in order: m_c and s_c are complete (all their live centre inputs are final), so
//      z_c = 0.1 m_c + exp(0.1 s_c) u_c; z_c's centre taps enter stage 0; then, stage by stage, the hidden units whose
//      last centre input was z_c are finalised (nonlinearity) and their centre taps enter the next stage.
// Which units become final at which step is derived on the host from iaf_tap_rule (iaf_capi.cu, inv_tables) and handed
// over as a table.  Each stage keeps a two-row ring of its input in shared memory (rows y and y+1, plus two zero pad
// columns); the weights are the SIMT pack (masked taps are zero) read through the read-only cache.
//
// Shared memory and __syncthreads only (no shuffles, no atomics, no scratch): the host emulation runs this kernel, and
// one sample's results are bit-identical whatever the batch.
#include "iaf_common.h"

#define IAF_INV_THREADS 128

__global__ void __launch_bounds__(IAF_INV_THREADS) iaf_inv_kernel(const __grid_constant__ IafInvParams p) {
  IAF_DYN_SMEM(float, smem);
  const int tid = threadIdx.x;
  const int n = blockIdx.x;
  const int H = p.H, W = p.W, HW = H * W, C = p.C, nst = p.n_stages, L = nst - 1;
  const int RP = W + 2;  // ring row pitch: columns -1 .. W
  float* lds = smem + p.lds_off;

  for (int i = tid; i < p.smem_floats; i += IAF_INV_THREADS) smem[i] = 0.f;
  __syncthreads();

  for (int y = H - 1; y >= 0; --y) {
    const int s0 = y & 1, s1 = s0 ^ 1;  // ring slots of rows y and y+1
    const bool byH = (y == H - 1);
    for (int x = W - 1; x >= 0; --x) {
      const bool bx0 = (x == 0), bxW = (x == W - 1);
      const int pix = y * W + x;
      const int gp = p.flip ? HW - 1 - pix : pix;

      // ---- 1. the non-centre taps of every stage ----
      {
        int j = 0, base = 0;
        for (int e = tid; e < p.n_units; e += IAF_INV_THREADS) {
          while (e >= base + p.stage[j].cout_pad) base += p.stage[j++].cout_pad;
          const IafStageDev& S = p.stage[j];
          const int col = e - base;
          if (j < L && col >= S.cout) continue;
          float v = __ldg(S.bias + col);
          if (S.padw) {  // pad channel = 1 where the tap falls outside the image (conv.py:77-83)
            if (bxW) v += __ldg(S.padw + col);
            if (byH || bx0) v += __ldg(S.padw + S.cout_pad + col);
            if (byH) v += __ldg(S.padw + 2 * S.cout_pad + col);
            if (byH || bxW) v += __ldg(S.padw + 3 * S.cout_pad + col);
          }
          if (j == 0 && L > 0) v += __ldg(p.ctx + ((size_t)n * S.cout + col) * HW + gp);  // ar.py:402 / layers.py:163
          const float* ring = smem + p.ring_off[j];
          const size_t ts = (size_t)S.cin * S.cout_pad;
          for (int ci = 0; ci < S.cin; ++ci) {
            const float* r0 = ring + (ci * 2 + s0) * RP + x + 1;
            const float* r1 = ring + (ci * 2 + s1) * RP + x + 1;
            const float* wc = S.w + (size_t)ci * S.cout_pad + col;
            v = fmaf(r0[1], __ldg(wc + ts), v);       // ( 0,+1)
            v = fmaf(r1[-1], __ldg(wc + 2 * ts), v);  // (+1,-1)
            v = fmaf(r1[0], __ldg(wc + 3 * ts), v);   // (+1, 0)
            v = fmaf(r1[1], __ldg(wc + 4 * ts), v);   // (+1,+1)
          }
          smem[p.acc_off[j] + col] = v;
        }
      }
      __syncthreads();

      // ---- 2. the chain over the z channels (step -1: the units that see no z channel at all) ----
      for (int k = -1; k < C; ++k) {
        if (k >= 0) {
          const int c = p.descending ? C - 1 - k : k;
          const int cm = (c >> 2) * 8 + (c & 3);  // heads interleaved in groups of 4 columns (iaf_pack.cu)
          const float* acch = smem + p.acc_off[L];
          const size_t g = ((size_t)n * C + c) * HW + gp;
          // the inverse of models.py:282-285: z = arw_mean + exp(arw_logsd) * u
          const float a = p.scale * acch[cm + 4];
          const float zc = fmaf(expf(a), __ldg(p.u + g), p.scale * acch[cm]);
          if (L == 0) __syncthreads();  // the heads are stage 0: m_c, s_c are read before z_c's taps are added
          if (tid == 0) {
            smem[p.ring_off[0] + (c * 2 + s0) * RP + x + 1] = zc;
            p.z_out[g] = zc;
            if (p.logsd_out) p.logsd_out[g] = a;
            lds[c] += a;
          }
          const IafStageDev& S = p.stage[0];
          const int nc = L ? S.cout : S.cout_pad;
          float* acc = smem + p.acc_off[0];
          const float* wc = S.w + (size_t)c * S.cout_pad;  // centre tap, input channel c
          for (int col = tid; col < nc; col += IAF_INV_THREADS) acc[col] = fmaf(__ldg(wc + col), zc, acc[col]);
          __syncthreads();
        }
        for (int j = 0; j < L; ++j) {
          const int* off = p.grp + p.grp_off[j];
          const int b0 = __ldg(off + k + 1), b1 = __ldg(off + k + 2);
          if (b0 == b1) continue;  // nothing of stage j became final: nothing later in this step either
          const int* units = off + C + 2;
          const float* acc = smem + p.acc_off[j];
          float* ring = smem + p.ring_off[j + 1];
          for (int i = b0 + tid; i < b1; i += IAF_INV_THREADS) {
            const int u = __ldg(units + i);
            ring[(u * 2 + s0) * RP + x + 1] = iaf_apply_nl(acc[u], p.nl);
          }
          __syncthreads();
          const IafStageDev& S = p.stage[j + 1];
          const int nc = (j + 1 < L) ? S.cout : S.cout_pad;
          float* nacc = smem + p.acc_off[j + 1];
          for (int col = tid; col < nc; col += IAF_INV_THREADS) {
            float v = nacc[col];
            for (int i = b0; i < b1; ++i) {
              const int u = __ldg(units + i);
              v = fmaf(__ldg(S.w + (size_t)u * S.cout_pad + col), ring[(u * 2 + s0) * RP + x + 1], v);
            }
            nacc[col] = v;
          }
          __syncthreads();
        }
      }
    }
  }

  if (tid == 0 && p.logdet_out) {  // logdet = -sum arw_logsd, per channel over the pixels, then over the channels
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += lds[c];
    p.logdet_out[n] = -s;
  }
}

static cudaError_t iaf_inv_set_smem() { return iaf_smem_optin(iaf_inv_kernel); }

static cudaError_t iaf_launch_inv(const IafInvParams& p, int B, size_t smem_bytes, cudaStream_t stream) {
  IAF_LAUNCH(iaf_inv_kernel, B, IAF_INV_THREADS, smem_bytes, stream, p);
  return cudaGetLastError();
}

namespace {
struct IafInvRegister {
  IafInvRegister() { iaf_inv = IafInvKernel{iaf_launch_inv, iaf_inv_set_smem}; }
} iaf_inv_register;
}  // namespace
