// Layer-at-a-time tensor-core kernel (Hopper wgmma): one launch per conv stage of the stack.  Included by iaf_tc.cu.
//
// Same slot-stream / implicit-GEMM formulation and fp16 hi/lo operand split as described there, and
//   * the stage's input operand comes from HBM/L2: either fp32 z (first stage, split on the fly by the worker warps into
//     a shared-memory A window) or the previous stage's output, stored as pre-split fp16 "operand images"
//     [channel chunk][slot][8] (hi and lo), so that a tile's A chunk pair is a few contiguous runs that the producer warp
//     fetches with 1-D bulk copies;
//   * the weights are NOT resident (unless they fit the ring): the producer warp streams them in chunks of LY_KC
//     K-steps through an NB-deep shared-memory ring (cp.async.bulk + expect_tx on an mbarrier); both MMA warpgroups
//     release a ring stage once their wgmma reads of it have completed;
//   * five warpgroups with their own jobs: warpgroups 0 and 1 issue the MMAs, warpgroup r for rows [64 r, +64) of the
//     tile and ALL of the stage's columns (one wgmma m64nNk16 per K-step, tap and product; two of half the width for
//     stages of 129-160 columns; two passes over K for 161-192), accumulating in registers; warpgroups 2 and 3 build the first stage's z window and
//     run the epilogues; in warpgroup 4, warp 16 is the producer and warp 17 the reducer.  setmaxnreg moves registers
//     from warpgroup 4 to the MMA warpgroups;
//   * the accumulators go through a shared-memory tile [128][N + 4] so that the epilogue keeps one thread per slot
//     (coalesced global traffic along pixels).  The tile, the z window and the fused kernel's hidden operand buffer
//     are handed between the MMA and epilogue warpgroups through full / empty mbarrier pairs, so an epilogue runs
//     while the MMAs of the next tile (or stage) are in flight: the MMA warpgroups' registers are the second buffer;
//   * hidden stages write their output operand image back to global memory (16-byte stores), the heads stage applies
//     the affine update; per-sample sums go through the reducer warp in fixed order.
#pragma once

#define LY_MMA_WARPS 8                   // warpgroups 0, 1: the MMAs
#define LY_EPI_WARP0 8                   // warpgroups 2, 3: z window and epilogues
#define LY_EPI_WARPS 8
#define LY_ETHREADS (LY_EPI_WARPS * 32)
#define LY_TMA_WARP 16                   // warpgroup 4: the producer, the reducer and two idle warps
#define LY_RED_WARP 17
#define LY_THREADS 640
// registers per thread after setmaxnreg.  The launch gives each of the 640 threads 96 (61,440 in all); warpgroup 4
// returns 48 of them and the MMA warpgroups take 24 more, for up to 80 accumulators (64 x 160 fp32 over 128 threads, or
// 2 x 64 x 64 when the correction products are summed apart) beside their descriptors and counters.  The epilogue
// warpgroups keep 96.  ptxas compiles the code after setmaxnreg.inc to the raised count, but each single wgmma must
// still fit the launch's 96: hence two instructions of half the width for 160 columns (ly_mma_tile).  96 accumulators
// (a 192-column span) do not fit in 120: stages of 161-192 columns run two passes over K of 96 columns each.
#define LY_REGS_AUX 48
#define LY_REGS_MMA 120
// per-sample partials of one tile (step and multiconv modes): one per (set of column groups g with the same g % 4,
// quarter of the tile's slots), summed by the reducer warp in that fixed order
#define LY_PART_SETS 16
#define LY_KC 5        // K-steps (of 16) per weight chunk
#define LY_MAX_NB 6
// Bytes every layout of the stage kernel reserves past its last weight image: the column span of an MMA warpgroup (see
// ly_mma_tile), 32 NGW columns, of the last K plane reads up to 16 * (32 * NGW - N) bytes past the plane's end -- 256 for
// the per-stage instantiations (NGW = ceil(N / 32)), 768 for the fused one (NGW = 2, N down to 16: hidden [16]) -- and
// that read must stay inside the CTA's allocation.  (The previous layout's second column half ended at the same byte.)
#define LY_B_SLACK 1024

enum { LB_BFULL = 0, LB_BEMPTY = LY_MAX_NB, LB_PART = 2 * LY_MAX_NB,
       LB_PART_EMPTY = 2 + 2 * LY_MAX_NB,  // + tile parity: the reducer warp has consumed the partials
       // MMA <-> epilogue handoffs, one phase per use (parity = use & 1): the accumulator tile (written by the MMA warps,
       // read by the epilogue warps), the z window (written by the epilogue warps, read by the MMA warpgroups) and the
       // fused kernel's hidden operand buffer (likewise)
       LB_ACC_FULL = 4 + 2 * LY_MAX_NB, LB_ACC_EMPTY, LB_WIN_FULL, LB_WIN_EMPTY, LB_H_FULL, LB_H_EMPTY,
       LB_COUNT };

struct IafLyParams {
  IafTcParams t;               // geometry, pointers, slot decoding (t.st[0] describes THIS stage)
  const __nv_bfloat16* a_hi;   // input operand image (in_mode 1)
  const __nv_bfloat16* a_lo;
  __nv_bfloat16* o_hi;         // output operand image (hidden stages)
  __nv_bfloat16* o_lo;
  int S_pad;                   // slots per chunk plane of the global images
  int in_mode;                 // 0: fp32 z (first stage), 1: operand image
  int is_heads;                // 1: last stage
  int first;                   // 1: first stage (adds the context)
  int NB;                      // weight ring depth
  int sm_a, sm_b, sm_bias, sm_part, sm_acc;
  int stage_bytes;             // bytes of one ring stage: 2 * b_chunk_bytes (+ 4 * WIN * 16 when the A pair rides along)
  int b_chunk_bytes;           // bytes of one ring slot half (hi or lo): LY_KC * 2 * N * 16
  int n_bchunks;               // weight chunks per tile
  int tl_enable;               // timeline builds only: this launch flushes its events
  // one-launch step for stacks with one hidden layer (the FUSED instantiation): t.st[0] is the hidden layer, t.st[1] the
  // heads; both weight images are resident, the hidden activations stay in shared memory
  int TS;                      // slots a tile advances: TC_TILE, or TC_TILE - MIR when fused (overlapped windows)
  int TO;                      // rows of a tile that produce outputs (TC_TILE, or TS when fused)
  int sm_h;                    // fused: the hidden operand buffer [chunk][TC_TILE + MIR][8] hi, then lo
  int sm_b1, sm_bias1;         // fused: the heads' resident weights and bias table
  int n_bchunks1, b_chunk_bytes1;
  // data-gradient use of a hidden stage (iaf_dg_run): the input image holds the gradient at this layer's output, scaled
  // per sample into fp16 range; weights are the transposed effective weights; t.ctx points at the activations h whose
  // nl' multiplies the result (bwd 1) or is null (bwd 2: gradient at the stack input, ACCUMULATED into hid_out)
  int bwd;                     // 0 forward, 1 x nl'(h), 2 identity and accumulate
  const float* amax;           // [B] per-sample max |gradient at the heads| (the scale is 2^(5 - floor(log2 amax)))
  const float* wscale;         // the power of two the stage's weight images carry (iaf_dg_wscale_kernel), undone here
};

// floats per row of the shared-memory accumulator tile: N + 4 keeps a warp's 16-byte row reads conflict-free
__host__ __device__ __forceinline__ int ly_acc_pitch(int N) { return N + 4; }

// nl'(pre-activation) from the activation h = nl(pre-activation)   (same table as iaf_bwd.cu's bw_nl_grad)
__device__ __forceinline__ float dg_nl_grad(float h, int nl) {
  switch (nl) {
    case IAF_NL_ELU: return h > 0.f ? 1.f : h + 1.f;
    case IAF_NL_SOFTPLUS: return 1.f - __expf(-h);
    case IAF_NL_RELU: return h > 0.f ? 1.f : 0.f;
    case IAF_NL_TANH: return 1.f - h * h;
    case IAF_NL_LEAKYRELU: return h < 0.f ? 0.01f : 1.f;
    default: return 1.f;
  }
}
// power-of-two scale that brings a sample's gradient into [32, 64): exact to apply and to undo
__device__ __forceinline__ float dg_scale_from_amax(float amax) {
  if (!(amax > 1e-30f) || !(amax < 1e30f)) return 1.0f;
  const int e = (int)((__float_as_uint(amax) >> 23) & 0xffu) - 127;  // floor(log2(amax)) for normal numbers
  return __uint_as_float((uint32_t)(127 + 5 - e) << 23);
}

// The MMAs of one stage (or one pass over it) for one tile, run by the two MMA warpgroups.  Warpgroup r computes rows
// [64 r, +64) and the 16 SPG columns from col0: D[64 x 16 SPG] += A_t[64 x 16] B_t[16 x 16 SPG] over K-steps, taps and
// the three split products, accumulating in registers (acc; returned with the correction sum added).  Each product is
// one wgmma over the span (NI = 1), or for 160 columns two of half the span (NI = 2): an m64n160 instruction needs more
// registers than the launch's 96 by itself, although all 80 accumulators fit after setmaxnreg.  The halves' fragments sit
// side by side in acc exactly as one instruction's would.  In the B image [K/8][N][8] a span of contiguous columns is one
// K-major descriptor (8-column groups 128 B apart, the two K halves one plane apart).  NGW is a compile-time count: a span
// past the stage's columns computes on whatever follows in shared memory -- the next K plane, the next image, or the
// LY_B_SLACK bytes every layout reserves past its last one -- and is not stored, so every wgmma is issued
// unconditionally and ptxas keeps them asynchronous.
//   ring: the tile's weight chunks are the CTA's gchunk, gchunk + 1, ... (every tile streams all n_chunks); chunk g sits
//   in ring stage g % NB (parity from g / NB), released after its MMAs complete;
//   otherwise resident: chunk c sits in stage c behind barrier bar0 + c (parity 0).
//   a_in_stage: the A chunk pair of K-step c rides in the ring stage before the weights; otherwise A is a window at a_addr,
//   and barrier a_release (if >= 0) is arrived on once the MMAs have read it.
// the two MMA warpgroups converge here before a stage's MMAs: without a barrier between the per-thread mbarrier waits
// and the accumulator set-up, ptxas treats the wgmma sequence as divergent code and serializes every wgmma
__device__ __forceinline__ void mma_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(LY_MMA_WARPS * 32) : "memory"); }

template <int SPG, bool SPLIT>
__device__ __forceinline__ void ly_mma_tile(float* acc, uint64_t* bars, int N, int col0, int n_chunks, bool ring, int NB,
                                            int gchunk, int bar0, uint32_t b_addr0, uint32_t stage_bytes,
                                            uint32_t b_chunk_bytes, bool a_in_stage, uint32_t a_addr, uint32_t a_plane,
                                            uint32_t a_lo_off, int Wp, int a_release) {
  constexpr int NA = 8 * SPG;          // accumulators per thread: 64 x 16 SPG over the 128 threads of the warpgroup
  constexpr int NI = SPG > 8 ? 2 : 1;  // wgmma instructions per product
  constexpr int GI = SPG / NI;         // 16-column groups per instruction
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rh = warp >> 2, wl = warp & 3;
  const uint32_t b_plane = (uint32_t)N * 16u;
  const uint32_t sh[IAF_NTAPS] = {0u, 1u, (uint32_t)(Wp - 1), (uint32_t)Wp, (uint32_t)(Wp + 1)};  // 16-byte units
  const uint32_t a_kstep = (2u * a_plane) >> 4, b_tstep = (2u * b_plane) >> 4;
  const uint32_t a_row = (uint32_t)(rh * 64);  // 64 slots = 64 descriptor units
  // The two correction products (lo x hi, hi x lo: 2^-11 of hi x hi) go to their own accumulators where registers allow:
  // added one by one to the main sum, each is rounded at the main sum's magnitude by the tensor cores' accumulation, and
  // over K = 160 those roundings reach ~2e-7 of a unit pre-activation -- enough to put a ReLU's derivative on the wrong
  // side of a pre-activation that small.  Summed apart and added once at the end, they cost one rounding.  Stages of at
  // most 64 columns do so.
  float acl[SPLIT ? NA : 1];
#pragma unroll
  for (int e = 0; e < NA; ++e) {
    acc[e] = 0.f;
    if (SPLIT) acl[SPLIT ? e : 0] = 0.f;
  }
  float* corr = SPLIT ? acl : acc;
  int prev_stg = -1;
  for (int c = 0; c < n_chunks; ++c) {
    const int stg = ring ? (int)((uint32_t)gchunk % (uint32_t)NB) : c;
    mbar_wait(&bars[bar0 + stg], ring ? ((uint32_t)gchunk / (uint32_t)NB) & 1u : 0u);
    const uint32_t sbase = b_addr0 + (uint32_t)stg * stage_bytes;
    uint32_t ah0, al0, bbase;
    if (a_in_stage) {
      ah0 = wg_desc_lo(sbase, a_plane);
      al0 = wg_desc_lo(sbase + 2u * a_plane, a_plane);
      bbase = sbase + 4u * a_plane;
    } else {
      ah0 = wg_desc_lo(a_addr, a_plane) + (uint32_t)c * a_kstep;
      al0 = wg_desc_lo(a_addr + a_lo_off, a_plane) + (uint32_t)c * a_kstep;
      bbase = sbase;
    }
    ah0 += a_row; al0 += a_row;
    const uint32_t bh0 = wg_desc_lo(bbase, b_plane) + (uint32_t)col0;  // 16 B per column
    const uint32_t bl0 = wg_desc_lo(bbase + b_chunk_bytes, b_plane) + (uint32_t)col0;
    wgmma_fence();
#pragma unroll 1
    for (int t = 0; t < IAF_NTAPS; ++t) {
      const uint64_t ah = mk_desc(ah0 + sh[t]), al = mk_desc(al0 + sh[t]);
      const uint32_t bt = (uint32_t)t * b_tstep;
#pragma unroll
      for (int h = 0; h < NI; ++h) {  // instruction h: columns [16 GI h, +16 GI), 16 B per column in the descriptor
        const uint32_t bc = bt + (uint32_t)(16 * GI * h);
        wgmma_m64nNk16<GI>(corr + 8 * GI * h, al, mk_desc(bh0 + bc));
        wgmma_m64nNk16<GI>(corr + 8 * GI * h, ah, mk_desc(bl0 + bc));
        wgmma_m64nNk16<GI>(acc + 8 * GI * h, ah, mk_desc(bh0 + bc));
      }
    }
    wgmma_commit();
    // keep this K-step's group in flight; the previous one has completed, so its ring stage can be refilled
    wgmma_wait<1>();
    if (ring && prev_stg >= 0 && wl == 0 && lane == 0) mbar_arrive(&bars[LB_BEMPTY + prev_stg]);
    prev_stg = stg;
    if (ring) ++gchunk;
  }
  wgmma_wait<0>();
  if (wl == 0 && lane == 0) {
    if (ring && prev_stg >= 0) mbar_arrive(&bars[LB_BEMPTY + prev_stg]);
    if (a_release >= 0) mbar_arrive(&bars[a_release]);
  }
  if (SPLIT) {
#pragma unroll
    for (int e = 0; e < NA; ++e) acc[e] += acl[SPLIT ? e : 0];
  }
}

// The MMA warpgroups' fragments -> columns [col0, +16 SPG) of the accumulator tile, for its k-th use in this launch: the
// first pass waits until the epilogue warps have read use k - 1, the last hands use k over.  acc[4j + 2h + e] = row
// 64 r + 16 wl + lane / 4 + 8h, column col0 + 8j + 2 (lane % 4) + e.
template <int SPG>
__device__ __forceinline__ void ly_acc_store(const float* acc, uint64_t* bars, float* s_acc, int N, int col0, int k,
                                             bool first, bool last) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (first && k >= 1) mbar_wait(&bars[LB_ACC_EMPTY], (uint32_t)((k - 1) & 1));
  const int pitch = ly_acc_pitch(N);
  const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < 2 * SPG; ++j) {
    const int c8 = col0 + 8 * j;
    if (c8 < N) {
      const int col = c8 + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(s_acc + (r0 + 8 * h) * pitch + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
  if (!last) return;
  __syncwarp();
  if (lane == 0) mbar_arrive(&bars[LB_ACC_FULL]);
}

// NGW: ceil(N / 32); an MMA warpgroup covers the stage's columns as 2 NGW groups of 16.  FUSED: the whole step of a one-hidden-layer stack in one
// launch (NGW covers both stages), tiles of TS = TC_TILE - MIR output slots whose 128 hidden rows overlap the next tile's.
template <bool PADW, int MODE, int NLT, int NGW, bool FUSED>
__global__ void __launch_bounds__(LY_THREADS, 1) iaf_ly_kernel(const __grid_constant__ IafLyParams q) {
  const IafTcParams& p = q.t;
  const int HW = p.HW;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[LB_COUNT];
  TL_DECL

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const IafTcStage& St0 = p.st[0];
  const int nchunk = St0.cin >> 3;
  const int a_plane = p.WIN * 16;          // bytes per chunk plane of the A window
  const int a_lo_off = nchunk * a_plane;
  // tiles of this CTA: u = blockIdx.x + i * gridDim.x
  const int n_my = (int)((uint32_t)(p.NT - (int)blockIdx.x + (int)gridDim.x - 1) / gridDim.x);
  const bool resident = FUSED || q.n_bchunks <= q.NB;
  const bool ring = !resident || q.in_mode;
  // an MMA warpgroup's span: all 32 NGW columns, or for NGW = 6 two passes over K of 96 columns each (the ring streams
  // the tile's chunks once per pass)
  constexpr int NP = NGW > 5 ? 2 : 1;
  constexpr int SPG = 2 * NGW / NP;
  constexpr bool SPLIT = NGW <= 2;

  // programmatic dependent launch: everything up to the barrier init overlaps the previous grid
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const bool epi = warp >= LY_EPI_WARP0 && warp < LY_EPI_WARP0 + LY_EPI_WARPS;
  const int et = tid - LY_EPI_WARP0 * 32, ew = warp - LY_EPI_WARP0;  // epilogue thread / warp index
  if (warp == LY_TMA_WARP) {
    if (lane == 0) {
      for (int i = 0; i < 2; ++i) {
        mbar_init(&bars[LB_PART + i], LY_EPI_WARPS);
        mbar_init(&bars[LB_PART_EMPTY + i], 1);
      }
      for (int i = 0; i < LY_MAX_NB; ++i) {
        mbar_init(&bars[LB_BFULL + i], 1);
        mbar_init(&bars[LB_BEMPTY + i], 2);  // both MMA warpgroups release the stage
      }
      mbar_init(&bars[LB_ACC_FULL], LY_MMA_WARPS);
      mbar_init(&bars[LB_ACC_EMPTY], LY_EPI_WARPS);
      mbar_init(&bars[LB_WIN_FULL], LY_EPI_WARPS);
      mbar_init(&bars[LB_WIN_EMPTY], 2);
      mbar_init(&bars[LB_H_FULL], LY_EPI_WARPS);
      mbar_init(&bars[LB_H_EMPTY], 2);
      fence_barrier_init();
    }
  } else if (epi) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int s = 0; s < (FUSED ? 2 : 1); ++s) {
      const IafTcStage& S = p.st[s];
      float* tb = reinterpret_cast<float*>(smem + (s ? q.sm_bias1 : q.sm_bias));
      for (int i = et; i < 5 * S.N; i += LY_ETHREADS) {
        float v = 0.f;
        if (i < S.N) v = __ldg(S.bias + i);
        else if (PADW) v = __ldg(S.padw + (i - S.N));
        tb[i] = v;
      }
    }
  }
  if (!epi) asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();

  if (warp >= LY_TMA_WARP) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(LY_REGS_AUX));
    if (warp == LY_TMA_WARP) {
      // ===================== producer: A windows (operand-image input) and the weight ring =====================
      if (lane == 0 && FUSED) {
        // both stages' weights, resident: hidden chunk c behind barrier c, heads chunk c behind barrier n_bchunks + c
        for (int s = 0; s < 2; ++s) {
          const IafTcStage& S = p.st[s];
          const int nb = s ? q.n_bchunks1 : q.n_bchunks, bcb = s ? q.b_chunk_bytes1 : q.b_chunk_bytes;
          uint8_t* base = smem + (s ? q.sm_b1 : q.sm_b);
          for (int c = 0; c < nb; ++c) {
            uint64_t* bar = &bars[LB_BFULL + (s ? q.n_bchunks : 0) + c];
            const size_t bo = (size_t)c * bcb;
            mbar_expect_tx(bar, (uint32_t)(2 * bcb));
            bulk_g2s(base + 2 * c * bcb, reinterpret_cast<const uint8_t*>(S.whi) + bo, (uint32_t)bcb, bar);
            bulk_g2s(base + 2 * c * bcb + bcb, reinterpret_cast<const uint8_t*>(S.wlo) + bo, (uint32_t)bcb, bar);
          }
        }
      } else if (lane == 0) {
        int gchunk = 0;
        for (int i = 0; i < n_my; ++i) {
          const int u = (int)blockIdx.x + i * (int)gridDim.x;
          // K order is [K-step within a tap][tap]: weight chunk c and A chunk pair (2c, 2c+1) are consumed together,
          // so both stream through shared memory at the pace of the MMAs
          for (int cp = 0; cp < (ring ? NP : 1) * q.n_bchunks; ++cp) {
            if (resident && i >= 1 && !q.in_mode) continue;  // weights already resident, A comes from the epilogue warps
            const int c = cp % q.n_bchunks;
            const int stg = gchunk % q.NB;
            const int use = gchunk / q.NB;
            if (use >= 1) {
              TL(2, 60, gchunk);
              mbar_wait(&bars[LB_BEMPTY + stg], (uint32_t)((use - 1) & 1));
              TL(2, 61, gchunk);
            }
            uint8_t* dst = smem + q.sm_b + stg * q.stage_bytes;
            const size_t bo = (size_t)c * q.b_chunk_bytes;
            if (q.in_mode) {
              // one ring stage = A chunk pair (hi c0, hi c1, lo c0, lo c1) + the weight chunk (hi, lo) of K-step c
              mbar_expect_tx(&bars[LB_BFULL + stg], (uint32_t)(4 * a_plane + 2 * q.b_chunk_bytes));
  #pragma unroll
              for (int h = 0; h < 2; ++h) {
                const size_t go = ((size_t)(2 * c + h) * q.S_pad + (size_t)u * TC_TILE) * 8;
                bulk_g2s(dst + h * a_plane, q.a_hi + go, (uint32_t)a_plane, &bars[LB_BFULL + stg]);
                bulk_g2s(dst + (2 + h) * a_plane, q.a_lo + go, (uint32_t)a_plane, &bars[LB_BFULL + stg]);
              }
              dst += 4 * a_plane;
            } else {
              mbar_expect_tx(&bars[LB_BFULL + stg], (uint32_t)(2 * q.b_chunk_bytes));
            }
            bulk_g2s(dst, reinterpret_cast<const uint8_t*>(St0.whi) + bo, (uint32_t)q.b_chunk_bytes, &bars[LB_BFULL + stg]);
            bulk_g2s(dst + q.b_chunk_bytes, reinterpret_cast<const uint8_t*>(St0.wlo) + bo, (uint32_t)q.b_chunk_bytes,
                     &bars[LB_BFULL + stg]);
            ++gchunk;
          }
        }
      }
      __syncwarp();
    } else if (warp == LY_RED_WARP && (FUSED || q.is_heads) && (p.persample_out || p.bc_out) && MODE != IAF_MODE_MULTICONV) {
      // ===================== reducer warp: per-tile partials -> per-sample outputs, off the workers' critical path ==========
      float* s_part = reinterpret_cast<float*>(smem + q.sm_part);
      constexpr bool LAY = (MODE == IAF_MODE_LAYER || MODE == IAF_MODE_LOGP);  // per-(sample, channel) partials
      for (int i = 0; i < n_my; ++i) {
        const int u = (int)blockIdx.x + i * (int)gridDim.x;
        const int pb = i & 1;
        const int tile_s0 = u * q.TS;
        const int n_first = fast_div(tile_s0, p.SPS, p.mg_sps);
        const int n_last = min(p.B - 1, fast_div(tile_s0 + q.TS - 1, p.SPS, p.mg_sps));
        const int ns = (tile_s0 < p.S) ? (n_last - n_first + 1) : 0;
        {
              mbar_wait(&bars[LB_PART + pb], (uint32_t)((i >> 1) & 1));
              const int cred = LAY ? p.C : 1;
              for (int k_ = lane; k_ < ns * cred; k_ += 32) {
                float tot = 0.f;
                if (LAY) {
                  const int nl_ = k_ / p.C, c = k_ - nl_ * p.C;
                  for (int qq = 0; qq < 4; ++qq) tot += s_part[((pb * 4 + qq) * p.MAXS + nl_) * p.C + c];
                } else {
                  for (int w = 0; w < LY_PART_SETS; ++w) tot += s_part[(pb * LY_PART_SETS + w) * p.MAXS + k_];
                }
                p.tilepart[((size_t)u * p.MAXS) * cred + k_] = tot;
                __threadfence();
              }
              __syncwarp();
              for (int k_ = lane; k_ < ns; k_ += 32) {
                const int n = n_first + k_;
                const int a = n * p.SPS, bb = a + p.SPS - 1;
                const int ta = a / q.TS, tbk = bb / q.TS;
                const unsigned expected = (unsigned)(tbk - ta + 1);
                __threadfence();
                if (atomicAdd(p.counter + n, 1u) == expected - 1u) {
                  __threadfence();
                  p.counter[n] = 0u;
                  float cost = 0.f;
                  for (int c = 0; c < cred; ++c) {
                    float tot = 0.f;
                    for (int tt = ta; tt <= tbk; ++tt) {
                      const int nf = fast_div(tt * q.TS, p.SPS, p.mg_sps);
                      tot += __ldcg(p.tilepart + ((size_t)tt * p.MAXS + (n - nf)) * cred + c);
                    }
                    if (LAY && p.bc_out) p.bc_out[(size_t)n * p.C + c] = tot;
                    cost += tot;
                  }
                  if (p.persample_out) p.persample_out[n] = LAY ? cost : -cost;
                }
              }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars[LB_PART_EMPTY + pb]);
      }
    }
    // warps 18 and 19 have nothing to do: they wait at the closing barrier with their 40 registers
  } else if (warp < LY_MMA_WARPS) {
    // ===================== MMA warpgroups: a tile's MMAs run while the epilogue warps finish the previous one =======
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(LY_REGS_MMA));
    float acc[8 * SPG];
    const bool tl0 = warp == 0 && lane == 0;
    for (int i = 0; i < n_my; ++i) {
      if (!q.in_mode) mbar_wait(&bars[LB_WIN_FULL], (uint32_t)(i & 1));
      mma_bar_sync();
      if (tl0) TL(0, 15, i);
#pragma unroll 1
      for (int ps = 0; ps < NP; ++ps) {
        if (ps) mma_bar_sync();
        ly_mma_tile<SPG, SPLIT>(acc, bars, St0.N, 16 * SPG * ps, q.n_bchunks, ring, q.NB, (i * NP + ps) * q.n_bchunks,
                                LB_BFULL, smem_u32(smem + q.sm_b), (uint32_t)(FUSED ? 2 * q.b_chunk_bytes : q.stage_bytes),
                                (uint32_t)q.b_chunk_bytes, q.in_mode != 0, smem_u32(smem + q.sm_a), (uint32_t)a_plane,
                                (uint32_t)a_lo_off, p.Wp, (q.in_mode || ps + 1 < NP) ? -1 : (int)LB_WIN_EMPTY);
        if (tl0 && ps + 1 == NP) TL(0, 20, i);
        ly_acc_store<SPG>(acc, bars, reinterpret_cast<float*>(smem + q.sm_acc), St0.N, 16 * SPG * ps, FUSED ? 2 * i : i,
                          ps == 0, ps + 1 == NP);
      }
      if (tl0) TL(0, 21, i);
      if (FUSED) {
        const IafTcStage& St1 = p.st[1];
        const int h_plane = (TC_TILE + p.MIR) * 16;
        mbar_wait(&bars[LB_H_FULL], (uint32_t)(i & 1));
        mma_bar_sync();
        if (tl0) TL(0, 35, i);
        ly_mma_tile<SPG, SPLIT>(acc, bars, St1.N, 0, q.n_bchunks1, false, 1, 0, LB_BFULL + q.n_bchunks,
                                smem_u32(smem + q.sm_b1), (uint32_t)(2 * q.b_chunk_bytes1), (uint32_t)q.b_chunk_bytes1,
                                false, smem_u32(smem + q.sm_h), (uint32_t)h_plane, (uint32_t)((St1.cin >> 3) * h_plane),
                                p.Wp, LB_H_EMPTY);
        if (tl0) TL(0, 40, i);
        ly_acc_store<SPG>(acc, bars, reinterpret_cast<float*>(smem + q.sm_acc), St1.N, 0, 2 * i + 1, true, true);
        if (tl0) TL(0, 41, i);
      }
    }
  } else {
    // ===================== epilogue warps: (first stage) z -> operand window; epilogues =====================
    const int qd = ew & 3, cg = ew >> 2;  // quarter of the tile's slots, first of the column groups g = cg + CGS k
    constexpr int CGS = LY_EPI_WARPS / 4;
    // the step-mode partials keep one per (g % 4, quarter): each warp covers two of the four column-group sets
    static_assert(CGS == 2 && LY_PART_SETS == 4 * 2 * CGS, "per-sample partial sets and epilogue warps out of step");
    const int sl = qd * 32 + lane;
    float* s_part = reinterpret_cast<float*>(smem + q.sm_part);
    float* s_acc = reinterpret_cast<float*>(smem + q.sm_acc);
    // this thread's slot row of the accumulator tile, 16 columns from c0, times the columns' inverse weight scales
    // (exact: powers of two; wsinv null = unscaled images, the data gradient's)
    auto acc_ld16 = [&](int c0, uint32_t* r, int pitch, const float* wsinv) {
      const float4* s4 = reinterpret_cast<const float4*>(s_acc + sl * pitch + c0);
#pragma unroll
      for (int e4 = 0; e4 < 4; ++e4) {
        float4 v4 = s4[e4];
        if (wsinv) {
          const float4 w4 = __ldg(reinterpret_cast<const float4*>(wsinv + c0) + e4);
          v4.x *= w4.x; v4.y *= w4.y; v4.z *= w4.z; v4.w *= w4.w;
        }
        r[4 * e4] = __float_as_uint(v4.x); r[4 * e4 + 1] = __float_as_uint(v4.y);
        r[4 * e4 + 2] = __float_as_uint(v4.z); r[4 * e4 + 3] = __float_as_uint(v4.w);
      }
    };
    const int h_plane = (TC_TILE + p.MIR) * 16;  // fused: bytes per chunk plane of the hidden operand buffer

    // fp32 z -> fp16 hi/lo A window of this CTA's i-th tile, once the MMAs have read tile i - 1's; handed to the MMAs
    auto build_window = [&](int i) {
      if (i >= 1) mbar_wait(&bars[LB_WIN_EMPTY], (uint32_t)((i - 1) & 1));
      const int u = (int)blockIdx.x + i * (int)gridDim.x;
#pragma unroll
      for (int it = 0; it < TC_ZITEMS; ++it) {
        const int idx = et + it * LY_ETHREADS;
        if (idx < p.WIN * nchunk) {
          const int ch = fast_div(idx, p.WIN, p.mg_win);
          const int s_ = idx - ch * p.WIN;
          const SlotInfo si = decode_slot(p, u * q.TS + s_, HW);
          float v[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = 0.f;
          if (si.valid) {
            const size_t g = ((size_t)si.n * p.C + ch * 8) * HW + si.gp;
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = __ldg(p.z + g + (size_t)e * HW);
            if (MODE == IAF_MODE_LAYER) {
#pragma unroll
              for (int e = 0; e < 8; ++e)
                v[e] = fmaf(fast_exp(__ldg(p.post_logsd + g + (size_t)e * HW)), v[e], __ldg(p.post_mean + g + (size_t)e * HW));
            }
          }
          uint8_t* dst = smem + q.sm_a + ch * a_plane + s_ * 16;
          split_store8(v, dst, dst + a_lo_off);
        }
      }
      fence_proxy_async();  // generic-proxy stores -> the wgmma (async proxy) reads of the window
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[LB_WIN_FULL]);
      if (ew == 0 && lane == 0) TL(1, 10, i);
    };
    // this warp is done reading the accumulator tile
    auto acc_release = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[LB_ACC_EMPTY]);
    };

    if (!q.in_mode) build_window(0);

    for (int i = 0; i < n_my; ++i) {
      const int u = (int)blockIdx.x + i * (int)gridDim.x;
      // per stage: the next tile's window goes to the MMAs before this tile's epilogue, which then runs under them
      if (!FUSED && !q.in_mode && i + 1 < n_my) build_window(i + 1);
      // the accumulator tile's uses: one per tile, or (fused) 2i for the hidden stage and 2i + 1 for the heads
      mbar_wait(&bars[LB_ACC_FULL], FUSED ? 0u : (uint32_t)(i & 1));
      if (ew == 0 && lane == 0) TL(1, 25, i);
      const SlotInfo si_all = decode_slot(p, u * q.TS + sl, HW);
      const bool bx0 = (si_all.x == 0), bxW = (si_all.x == p.W - 1), byH = (si_all.y == p.H - 1);

      // hidden stage epilogue: the next operand (global image, or the fused kernel's shared-memory buffer)
      auto hidden_epi = [&](const IafTcStage& St, const float* tb, const int ngroups, const int pitch, const SlotInfo si) {
        auto store_operand = [&](const float* v8, int chunk) {
          if (FUSED) {
            uint8_t* dst = smem + q.sm_h + chunk * h_plane + sl * 16;
            split_store8(v8, dst, dst + (St.N >> 3) * h_plane);
          } else {
            const size_t go = ((size_t)chunk * q.S_pad + (size_t)u * TC_TILE + sl) * 8;
            split_store8(v8, reinterpret_cast<uint8_t*>(q.o_hi + go), reinterpret_cast<uint8_t*>(q.o_lo + go));
          }
        };
          // context of the NEXT column group is fetched while the current one is computed
          float cxn[16];
          auto fetch_ctx = [&](int g) {
            if (q.first && si.valid && g < ngroups) {  // += context   (ar.py:402 / layers.py:163)
              const float* cp = p.ctx + ((size_t)si.n * St.N + g * 16) * HW + si.gp;
  #pragma unroll
              for (int e = 0; e < 16; ++e) cxn[e] = __ldg(cp + (size_t)e * HW);
            } else {
  #pragma unroll
              for (int e = 0; e < 16; ++e) cxn[e] = 0.f;
            }
          };
          fetch_ctx(cg);
          for (int g = cg; g < ngroups; g += CGS) {
            const int c0 = g * 16;
            float cx[16];
  #pragma unroll
            for (int e = 0; e < 16; ++e) cx[e] = cxn[e];
            fetch_ctx(g + CGS);
            uint32_t r[16];
            acc_ld16(c0, r, pitch, St.wsinv);
            if (q.bwd) {
              // data gradient: acc = (c W)^T g (scaled units); / c (exact: a power of two), x nl'(h), evaluated from the
              // activation itself
              const float sc = si.valid ? dg_scale_from_amax(__ldg(q.amax + si.n)) : 1.0f;
              const float inv = 1.0f / sc;
              const float winv = 1.0f / __ldg(q.wscale);
              float vb[16];
  #pragma unroll
              for (int e = 0; e < 16; ++e) {
                const float a = __uint_as_float(r[e]) * winv;
                const float d = (q.bwd == 1) ? dg_nl_grad(cx[e], p.nl) : 1.0f;
                vb[e] = si.valid ? a * d : 0.f;
              }
              if (St.hid_out && si.valid && sl < q.TO && u < p.NT) {
                float* hp = St.hid_out + ((size_t)si.n * St.N + c0) * HW + si.gp;
                if (q.bwd == 2) {
  #pragma unroll
                  for (int e = 0; e < 16; ++e) hp[(size_t)e * HW] += vb[e] * inv;
                } else {
  #pragma unroll
                  for (int e = 0; e < 16; ++e) hp[(size_t)e * HW] = vb[e] * inv;
                }
              }
              if (u < p.NT && q.o_hi) {
  #pragma unroll
                for (int hch = 0; hch < 2; ++hch) {
                  store_operand(vb + 8 * hch, (c0 >> 3) + hch);
                }
              }
              continue;
            }
            float v[16];
            {
              // branch-free: bias rows come in as 16-byte vectors, the pad-channel terms (conv.py:77-83: the pad
              // channel is 1 where a tap falls outside the image) are 0/1-weighted FMAs, and an invalid slot
              // (pad column, zero row, past the end) is selected to zero: that zero IS the conv's padding.  A select, not
              // a multiply: the zero row of sample n - 1 is computed from row 0 of sample n (every tap shift is
              // forward), and NaN * 0 would carry a non-finite sample n into its neighbour's outputs
              const float4* tb4 = reinterpret_cast<const float4*>(tb + c0);
              float bsv[16];
  #pragma unroll
              for (int e4 = 0; e4 < 4; ++e4) {
                const float4 t4 = tb4[e4];
                bsv[4 * e4] = t4.x; bsv[4 * e4 + 1] = t4.y; bsv[4 * e4 + 2] = t4.z; bsv[4 * e4 + 3] = t4.w;
              }
              if (PADW) {
                const float f1 = bxW ? 1.f : 0.f, f2 = (byH || bx0) ? 1.f : 0.f, f3 = byH ? 1.f : 0.f,
                            f4 = (byH || bxW) ? 1.f : 0.f;
  #pragma unroll
                for (int e = 0; e < 16; ++e)
                  bsv[e] += f1 * tb[St.N + c0 + e] + f2 * tb[2 * St.N + c0 + e] + f3 * tb[3 * St.N + c0 + e] +
                            f4 * tb[4 * St.N + c0 + e];
              }
  #pragma unroll
              for (int e = 0; e < 16; ++e) {
                const float a = __uint_as_float(r[e]) + bsv[e] + cx[e];
                float o;
                if (NLT == IAF_NL_ELU) {
                  const float ex = fast_exp(fminf(a, 0.f)) - 1.0f;  // elu, exp always evaluated: no divergence
                  o = a < 0.f ? ex : a;
                } else {
                  o = tc_apply_nl<NLT>(a, p.nl);
                }
                v[e] = si.valid ? o : 0.f;
              }
            }
            if (St.hid_out && si.valid && sl < q.TO && u < p.NT) {  // training forward: keep the activations for iaf_step_bwd_saved
              float* hp = St.hid_out + ((size_t)si.n * St.N + c0) * HW + si.gp;
  #pragma unroll
              for (int e = 0; e < 16; ++e) hp[(size_t)e * HW] = v[e];
            }
            if (u < p.NT) {
  #pragma unroll
              for (int hch = 0; hch < 2; ++hch) {
                store_operand(v + 8 * hch, (c0 >> 3) + hch);
              }
            }
          }
      };
      // heads epilogue: affine update, per-element and per-sample outputs
      auto heads_epi = [&](const IafTcStage& St, const float* tb, const int ngroups, const int pitch, const SlotInfo si) {
          // ---------------- heads: affine update, per-element and per-sample outputs ----------------
          // layer and logp modes: per-(sample, channel) partials, the 8 channels of a column group apart
          constexpr bool PERCH = (MODE == IAF_MODE_LAYER || MODE == IAF_MODE_LOGP);
          constexpr int NRED = PERCH ? 8 : 1;
          float red[NRED];
  #pragma unroll
          for (int k_ = 0; k_ < NRED; ++k_) red[k_] = 0.f;
          // step mode: the running sums of this thread's two column-group sets g % 4 = cg and cg + 2 (red[0] holds
          // the current group's set while it is summed), so each partial adds the same terms in the same order as
          // one warp per set would
          float rs0 = 0.f, rs1 = 0.f;
          const int tile_s0 = u * q.TS;
          const int n_first = fast_div(tile_s0, p.SPS, p.mg_sps);
          const int n_last = min(p.B - 1, fast_div(tile_s0 + q.TS - 1, p.SPS, p.mg_sps));
          const int ns = (tile_s0 < p.S) ? (n_last - n_first + 1) : 0;
          const int pb = i & 1;
          if (PERCH && (p.persample_out || p.bc_out) && i >= 2)
            mbar_wait(&bars[LB_PART_EMPTY + pb], (uint32_t)(((i >> 1) - 1) & 1));
          for (int g = cg; g < ngroups; g += CGS) {
            const int c0 = g * 16;
            const int ch0 = g * 8;
            float zv[8];
            size_t gi = 0;
            if (si.valid) {
              gi = ((size_t)si.n * p.C + ch0) * HW + si.gp;
  #pragma unroll
              for (int e = 0; e < 8; ++e) zv[e] = __ldg(p.z + gi + (size_t)e * HW);
            }
            uint32_t r[16];
            acc_ld16(c0, r, pitch, St.wsinv);
            const bool set_hi = ((g - cg) / CGS) & 1;
            if (PERCH) {
  #pragma unroll
              for (int k_ = 0; k_ < NRED; ++k_) red[k_] = 0.f;
            } else {
              red[0] = set_hi ? rs1 : rs0;
            }
            if (si.valid) {
  #pragma unroll
              for (int e = 0; e < 8; ++e) {
                float m = __uint_as_float(r[e]) + tb[c0 + e];
                float sv = __uint_as_float(r[8 + e]) + tb[c0 + 8 + e];
                if (PADW) {
                  if (bxW) { m += tb[St.N + c0 + e]; sv += tb[St.N + c0 + 8 + e]; }
                  if (byH || bx0) { m += tb[2 * St.N + c0 + e]; sv += tb[2 * St.N + c0 + 8 + e]; }
                  if (byH) { m += tb[3 * St.N + c0 + e]; sv += tb[3 * St.N + c0 + 8 + e]; }
                  if (byH || bxW) { m += tb[4 * St.N + c0 + e]; sv += tb[4 * St.N + c0 + 8 + e]; }
                }
                if (MODE == IAF_MODE_MULTICONV) {  // the un-fused operator: raw heads (ar.py:405-411 / layers.py:166)
                    p.z_out[gi + (size_t)e * HW] = m;
                    p.elem[gi + (size_t)e * HW] = sv;
                    continue;
                  }
                  const float arw_mean = p.scale * m, arw_logsd = p.scale * sv;  // models.py:282-285
                const size_t ge = gi + (size_t)e * HW;
                float z0 = zv[e];
                float eps = 0.f, pls = 0.f;
                if (MODE == IAF_MODE_LAYER) {
                  eps = z0;
                  pls = __ldg(p.post_logsd + ge);
                  z0 = fmaf(fast_exp(pls), eps, __ldg(p.post_mean + ge));
                }
                const float zn = (z0 - arw_mean) * fast_exp(-arw_logsd);
                if (MODE != IAF_MODE_LOGP || p.z_out) p.z_out[ge] = zn;
                if (MODE == IAF_MODE_LOGP) {
                  // MADE prior (models.py:304-309, rand.py:83): the standard normal at z', - arw_logsd
                  const float lp = -0.9189385332046727f - arw_logsd - 0.5f * zn * zn;
                  if (p.elem) p.elem[ge] = arw_logsd;
                  if (p.logps) p.logps[ge] = lp;
                  red[e] = lp;
                } else if (MODE == IAF_MODE_STEP) {
                  if (p.elem) p.elem[ge] = arw_logsd;
                  red[0] += arw_logsd;
                } else {
                  const float logqs = -0.9189385332046727f - pls - 0.5f * eps * eps + arw_logsd;
                  const float pl = __ldg(p.prior_logsd + ge);
                  const float d = zn - __ldg(p.prior_mean + ge);
                  const float logps = -0.9189385332046727f - pl - 0.5f * d * d * fast_exp(-2.0f * pl);
                  const float kl = logqs - logps;
                  if (p.elem) p.elem[ge] = kl;
                  red[e] = kl;
                }
              }
            }
            if (!PERCH) {
              if (set_hi) rs1 = red[0];
              else rs0 = red[0];
            }
            if (PERCH) {
              for (int nl_ = 0; nl_ < ns; ++nl_) {
  #pragma unroll
                for (int e = 0; e < 8; ++e) {
                  float x = (si.valid && si.n == n_first + nl_) ? red[e] : 0.f;
  #pragma unroll
                  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
                  if (lane == 0) s_part[((pb * 4 + qd) * p.MAXS + nl_) * p.C + ch0 + e] = x;
                }
              }
            }
          }

          if (p.persample_out || p.bc_out) {
            if (!PERCH) {
              if (i >= 2) mbar_wait(&bars[LB_PART_EMPTY + pb], (uint32_t)(((i >> 1) - 1) & 1));
              for (int nl_ = 0; nl_ < ns; ++nl_) {
  #pragma unroll
                for (int h2 = 0; h2 < 2; ++h2) {
                  float x = (si.valid && si.n == n_first + nl_) ? (h2 ? rs1 : rs0) : 0.f;
  #pragma unroll
                  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
                  if (lane == 0) s_part[(pb * LY_PART_SETS + (cg + CGS * h2) * 4 + qd) * p.MAXS + nl_] = x;
                }
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bars[LB_PART + pb]);
          }
      };

      const float* tb0 = reinterpret_cast<const float*>(smem + q.sm_bias);
      if (FUSED) {
        // the hidden epilogue refills the hidden operand buffer once the heads MMAs of tile i - 1 have read it
        if (i >= 1) mbar_wait(&bars[LB_H_EMPTY], (uint32_t)((i - 1) & 1));
        hidden_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), si_all);
        fence_proxy_async();  // generic-proxy stores -> the heads' wgmma reads of the buffer
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars[LB_H_FULL]);
        acc_release();
        if (ew == 0 && lane == 0) TL(1, 30, i);
        // the next tile's window is built under the heads MMAs, the heads epilogue runs under the next hidden MMAs
        if (i + 1 < n_my) build_window(i + 1);
        mbar_wait(&bars[LB_ACC_FULL], 1u);
        if (ew == 0 && lane == 0) TL(1, 45, i);
        const IafTcStage& St1 = p.st[1];
        SlotInfo si_out = si_all;
        si_out.valid = si_all.valid && sl < q.TO;
        heads_epi(St1, reinterpret_cast<const float*>(smem + q.sm_bias1), St1.N >> 4, ly_acc_pitch(St1.N), si_out);
        acc_release();
        if (ew == 0 && lane == 0) TL(1, 50, i);
      } else {
        if (!q.is_heads) hidden_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), si_all);
        else heads_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), si_all);
        acc_release();
        if (ew == 0 && lane == 0) TL(1, 30, i);
      }
    }
  }

  __syncthreads();
  if (q.tl_enable) {
    if (tid == 0) TL(1, 98, MODE);
    if (tid == 0) TL(1, 99, n_my);
    __syncwarp();
    TL_FLUSH
  }
}
