// Weight gradient of one masked conv layer on the tensor cores (included by iaf_tc.cu).
//
//   dW[tap][ci][co] = sum over slots r of  X[r][ci] * G[r + shift_tap][co]          (point-reflected stream)
//
// X (the layer's input activations) and G (the gradient at its pre-activation output) are the SAME operand images the
// forward and the data gradient use -- [chunk of 8 channels][slot][8] fp16 hi / lo -- but read with the SLOT stream as
// K: 8 consecutive slots of a chunk plane are exactly one core matrix of the canonical no-swizzle MN-MAJOR layout
// (8 K-rows x 16 bytes of 8 contiguous channels), LBO = 128 B between K groups, SBO = the plane pitch between channel
// groups, and a tap is still `shift x 16` bytes on G's start address.  Both operands are MN-major (wgmma transpose
// flags).  Per tap and per 16 slots: D_tap[ci][co] += X^T G; two warpgroups of M = 64 input channels make a block of
// 128 (rows past the layer's channels read whatever follows in shared memory and are never stored), N = a part of the
// columns of at most 48 (5 taps x Np / 2 accumulator registers per thread), the same three split-operand products as
// everywhere (X_lo G_hi, X_hi G_lo, X_hi G_hi).  Layers of at most 64 input channels run one warpgroup per CTA.  The
// column groups (NGRP) and warpgroups (NWG) are compile-time counts, so no wgmma sits behind a run-time condition.
//
// Work split: one CTA per (channel block, column part, split-K group); the group walks K tiles of WG_KT slots through a
// bulk-copy ring; partial sums go to part[group][...] and the fixed-order reduction kernel of iaf_bwd.cu adds them.
// The images carry per-sample scales (s_n on G, c / s_n on X, c = the smallest s_n; see iaf_dg_image_kernel), so the
// product carries the single factor c, removed here.
#pragma once

#define WG_KT 64          // slots per K tile (4 MMAs of K = 16 per tap and product)
#define WG_HALO 24        // G slots past the tile a tap can reach (>= Wp + 1, multiple of 8)
#define WG_MAX_STAGES 6
#define WG_MAX_NP 48      // columns per CTA (5 taps x 24 accumulator registers per thread at most)
#define WG_THREADS(NWG) ((4 * (NWG) + 1) * 32)  // NWG consumer warpgroups of 64 input channels, one producer warp

struct IafWgTcParams {
  const __nv_bfloat16* x_hi;  // [x_planes/8][S_pad][8]
  const __nv_bfloat16* x_lo;
  const __nv_bfloat16* g_hi;  // [g_planes/8][S_pad][8]
  const __nv_bfloat16* g_lo;
  float* part;                // [NG][5 * cin * ncol (+ 5 * ncol unused here)]
  const float* amax;          // [B]: c = scale of the largest
  int B, cin, ncol, S_pad, Wp;
  int n_mb, n_np, Np;         // channel blocks of 128, column parts of Np
  int NTK, NG;                // K tiles in all, split-K groups
  int part_stride;            // floats per group in `part`
  int n_stages, stage_bytes, xa_bytes;  // ring: per stage [X hi planes][X lo planes][G hi planes][G lo planes]
  int xplanes, gplanes;       // chunk planes staged per tile: of this CTA's channel block / column part
};

template <int NGRP, int NWG>
__global__ void __launch_bounds__(WG_THREADS(NWG), 1) iaf_wg_kernel(const __grid_constant__ IafWgTcParams p) {
  constexpr int WG_CONS = 4 * NWG, WG_W_TMA = WG_CONS;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[2 * WG_MAX_STAGES];
  uint64_t* full = bars;
  uint64_t* empty = bars + WG_MAX_STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int bid = blockIdx.x;
  const int np = bid % p.n_np; bid /= p.n_np;
  const int mb = bid % p.n_mb;
  const int g = bid / p.n_mb;
  const int x_pitch = WG_KT * 16, g_pitch = (WG_KT + WG_HALO) * 16;  // bytes per chunk plane in a stage
  const int n_my = (p.NTK - g + p.NG - 1) / p.NG;                      // K tiles u = g, g + NG, ...
  const int xpl = min(p.xplanes, (p.cin >> 3) - mb * 16);               // chunk planes this channel block really has

  if (warp == WG_W_TMA && lane == 0) {
    for (int i = 0; i < WG_MAX_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], NWG);  // every consumer warpgroup releases a stage
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == WG_W_TMA) {
    // one bulk copy per chunk plane and image; the lanes of the warp issue them side by side
    const uint32_t tx = (uint32_t)(2 * xpl * x_pitch + 2 * p.gplanes * g_pitch);
    const int ncp = 2 * xpl + 2 * p.gplanes;
    for (int i = 0; i < n_my; ++i) {
      const int u = g + i * p.NG;
      const int stg = i % p.n_stages, use = i / p.n_stages;
      if (use >= 1) mbar_wait(&empty[stg], (uint32_t)((use - 1) & 1));
      uint8_t* dst = smem + (size_t)stg * p.stage_bytes;
      if (lane == 0) mbar_expect_tx(&full[stg], tx);
      __syncwarp();
      const size_t s0 = (size_t)u * WG_KT;
      for (int k = lane; k < ncp; k += 32) {
        if (k < 2 * xpl) {
          const int lo = k >= xpl, c = lo ? k - xpl : k;
          const size_t go = ((size_t)(mb * 16 + c) * p.S_pad + s0) * 8;
          bulk_g2s(dst + ((lo ? p.xplanes : 0) + c) * x_pitch, (lo ? p.x_lo : p.x_hi) + go, (uint32_t)x_pitch, &full[stg]);
        } else {
          const int kk = k - 2 * xpl;
          const int lo = kk >= p.gplanes, c = lo ? kk - p.gplanes : kk;
          const size_t go = ((size_t)(np * (p.Np >> 3) + c) * p.S_pad + s0) * 8;
          bulk_g2s(dst + p.xa_bytes + ((lo ? p.gplanes : 0) + c) * g_pitch, (lo ? p.g_lo : p.g_hi) + go, (uint32_t)g_pitch,
                   &full[stg]);
        }
      }
      __syncwarp();
    }
  } else if (warp < WG_CONS) {
    // consumer warpgroup wgi: input channels [64 wgi, +64) of the block, every column of the part, all five taps
    const int wgi = warp >> 2, wl = warp & 3;
    float* out = p.part + (size_t)g * p.part_stride;
    float acc[IAF_NTAPS][NGRP][8];
#pragma unroll
    for (int t = 0; t < IAF_NTAPS; ++t)
#pragma unroll
      for (int k = 0; k < NGRP; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[t][k][e] = 0.f;
    // high words: SBO = the plane pitch (next 8 channels); low words: start (16-byte units) | LBO = 128 B (next 8 slots)
    const uint32_t x_hi_w = (uint32_t)x_pitch >> 4, g_hi_w = (uint32_t)g_pitch >> 4;
    const uint32_t sh[IAF_NTAPS] = {0u, 1u, (uint32_t)(p.Wp - 1), (uint32_t)p.Wp, (uint32_t)(p.Wp + 1)};
    for (int i = 0; i < n_my; ++i) {
      const int stg = i % p.n_stages, use = i / p.n_stages;
      mbar_wait(&full[stg], (uint32_t)(use & 1));
      const uint32_t sbase = smem_u32(smem + (size_t)stg * p.stage_bytes);
      const uint32_t xh0 = wg_desc_lo(sbase + (uint32_t)(wgi * 8 * x_pitch), 128u);
      const uint32_t xl0 = wg_desc_lo(sbase + (uint32_t)((p.xplanes + wgi * 8) * x_pitch), 128u);
      const uint32_t gh0 = wg_desc_lo(sbase + (uint32_t)p.xa_bytes, 128u);
      const uint32_t gl0 = wg_desc_lo(sbase + (uint32_t)p.xa_bytes + (uint32_t)(p.gplanes * g_pitch), 128u);
      const uint32_t g_grp = (uint32_t)(2 * g_pitch) >> 4;  // 16 columns = two chunk planes
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < IAF_NTAPS; ++t) {
#pragma unroll
        for (int ks = 0; ks < WG_KT / 16; ++ks) {
          const uint32_t xo = (uint32_t)(ks * 16), go = (uint32_t)(ks * 16) + sh[t];  // 16-byte units = slots
          const uint64_t xh = ((uint64_t)x_hi_w << 32) | (xh0 + xo), xl = ((uint64_t)x_hi_w << 32) | (xl0 + xo);
#pragma unroll
          for (int k = 0; k < NGRP; ++k) {
            const uint32_t gk = go + (uint32_t)k * g_grp;
            const uint64_t gh = ((uint64_t)g_hi_w << 32) | (gh0 + gk), gl = ((uint64_t)g_hi_w << 32) | (gl0 + gk);
            wgmma_m64n16k16<1>(acc[t][k], xl, gh);
            wgmma_m64n16k16<1>(acc[t][k], xh, gl);
            wgmma_m64n16k16<1>(acc[t][k], xh, gh);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (wl == 0 && lane == 0) mbar_arrive(&empty[stg]);
    }
    // D_tap[ci][co] -> part[g][(tap * cin + ci) * ncol + co] / c
    float inv_c = 0.f;
    if (n_my > 0) {
      float am = 0.f;
      for (int n = 0; n < p.B; ++n) am = fmaxf(am, __ldg(p.amax + n));
      inv_c = 1.0f / dg_scale_from_amax(am);
    }
    const int ci0 = mb * 128 + wgi * 64 + wl * 16 + (lane >> 2);
#pragma unroll
    for (int t = 0; t < IAF_NTAPS; ++t)
#pragma unroll
      for (int k = 0; k < NGRP; ++k) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ci = ci0 + 8 * h;
          if (ci < p.cin) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const int co = np * p.Np + 16 * k + 8 * j + 2 * (lane & 3);
              *reinterpret_cast<float2*>(out + ((size_t)t * p.cin + ci) * p.ncol + co) =
                  make_float2(acc[t][k][4 * j + 2 * h] * inv_c, acc[t][k][4 * j + 2 * h + 1] * inv_c);
            }
          }
        }
      }
  }
}

typedef void (*WgKernel)(const IafWgTcParams);
// column groups of 16 per CTA (Np / 16) and consumer warpgroups (2 for layers of more than 64 input channels)
static WgKernel wg_kernel_pick(int ngrp, int nwg) {
  switch (ngrp * 2 + (nwg - 1)) {
    case 2: return iaf_wg_kernel<1, 1>;
    case 3: return iaf_wg_kernel<1, 2>;
    case 4: return iaf_wg_kernel<2, 1>;
    case 5: return iaf_wg_kernel<2, 2>;
    case 6: return iaf_wg_kernel<3, 1>;
    default: return iaf_wg_kernel<3, 2>;
  }
}
