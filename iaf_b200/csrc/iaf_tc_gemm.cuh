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
//     tile and ALL of the stage's columns (one wgmma m64nNk16 per K-step, tap and product; two per K-step and tap, the
//     second of twice the width, for spans of at most 64 columns; two of half the width for stages of 129-160 columns;
//     two passes over K for 161-192), accumulating in registers; warpgroups 2 and 3 run the epilogues; in warpgroup 4,
//     warp 16 is the producer, warp 17 the reducer and warps 18 and 19 build the first stage's z window.  setmaxnreg
//     moves registers from warpgroup 4 to the MMA warpgroups;
//   * the accumulators go through a shared-memory tile [128][N + 4] so that the epilogue keeps one thread per slot
//     (coalesced global traffic along pixels).  The tile, the z window and the fused kernel's hidden operand buffer
//     are handed between the MMA warpgroups and the warps that fill or drain them through full / empty mbarrier pairs,
//     so an epilogue runs while the MMAs of the next tile (or stage) are in flight: the MMA warpgroups' registers are the
//     second buffer.  The fused kernel's hidden buffer is handed over per 16-channel chunk, so the heads MMAs of a chunk
//     run while the hidden epilogue computes the later ones;
//   * hidden stages write their output operand image back to global memory (16-byte stores), the heads stage applies
//     the affine update; per-sample sums go through the reducer warp in fixed order.
#pragma once

#include <type_traits>

#define LY_MMA_WARPS 8                   // warpgroups 0, 1: the MMAs
#define LY_EPI_WARP0 8                   // warpgroups 2, 3: the epilogues
#define LY_EPI_WARPS 8
#define LY_ETHREADS (LY_EPI_WARPS * 32)
#define LY_TMA_WARP 16                   // warpgroup 4: the producer, the reducer and two window builders
#define LY_RED_WARP 17
#define LY_THREADS 640
// registers per thread after setmaxnreg.  The launch gives each of the 640 threads 96 (61,440 in all); warpgroup 4
// (producer, reducer, window builders) returns some of them to the MMA warpgroups, which hold up to 80 accumulators
// (64 x 160 fp32 over 128 threads) or 64 (2 x 64 x 64 when the correction products are summed apart) beside their
// descriptors and counters; the epilogue warpgroups keep 96.  Stages of 129-160 columns (NGW 5, 80 accumulators): MMA
// 112, warpgroup 4 64.  Every other instantiation (at most 64 accumulators): MMA 104, warpgroup 4 80, where the reducer
// and the window builders do not spill (at 48 the layer and logp variants spilled 12-44 B of stores).  Either way
// 256 x MMA + 128 x aux = 256 x 120 + 128 x 48.  ptxas compiles the code after setmaxnreg.inc to the raised count, but
// each single wgmma must still fit the launch's 96: hence two instructions of half the width for 160 columns
// (ly_mma_tile).  96 accumulators (a 192-column span) do not fit: stages of 161-192 columns run two passes over K of
// 96 columns each.
__host__ __device__ constexpr int ly_regs_mma(int ngw) { return ngw == 5 ? 112 : 104; }
__host__ __device__ constexpr int ly_regs_aux(int ngw) { return 48 + 2 * (120 - ly_regs_mma(ngw)); }
// per-sample partials of one tile (step and multiconv modes): one per (set of column groups g with the same g % 4,
// quarter of the tile's slots), summed by the reducer warp in that fixed order
#define LY_PART_SETS 16
#define LY_KC 5        // K-steps (of 16) per weight chunk
#define LY_MAX_NB 6
#define LY_H_CHUNKS 4  // fused: 16-channel chunks of the hidden operand buffer (hidden width <= 32 FZ_NGW = 64)
#define LY_WIN_WARP0 18  // warpgroup 4's last two warps build the first stage's z window
#define LY_WIN_WARPS 2
// Stages whose MMA warpgroup spans at most 32 LY_SPLIT_NGW columns (SPLIT, see ly_mma_tile) sum the correction products
// apart and keep their weights as one image [K/8][2 NS][8], NS = 32 NGW the span: each K plane holds the lo columns
// [0, NS), then the hi columns [NS, 2 NS), both halves zero from N on.  Wider stages keep a hi and a lo image [K/8][N][8].
#define LY_SPLIT_NGW 2
// Bytes every layout of the stage kernel reserves past its last weight image.  A SPLIT stage's spans end inside their K
// plane.  A wider stage's span, 32 NGW columns with NGW = ceil(N / 32), of the last K plane reads up to
// 16 * (32 * NGW - N) = 256 bytes past the plane's end, and that read must stay inside the CTA's allocation.  The
// reserve is kept at 1024 bytes, as when the one-launch kernel's spans could read 768 bytes past N = 16, so that every
// layout's size, and with it which stacks run in one launch, is unchanged.
#define LY_B_SLACK 1024

enum { LB_BFULL = 0, LB_BEMPTY = LY_MAX_NB, LB_PART = 2 * LY_MAX_NB,
       LB_PART_EMPTY = 2 + 2 * LY_MAX_NB,  // + tile parity: the reducer warp has consumed the partials
       // MMA <-> epilogue handoffs, one phase per use (parity = use & 1): the accumulator tile (written by the MMA warps,
       // read by the epilogue warps), the z window (written by the builder warps, read by the MMA warpgroups) and the
       // fused kernel's hidden operand buffer (written by the epilogue warps, read by the MMA warpgroups): full per
       // 16-channel chunk c, LB_H_FULL + c, so that the heads MMAs of chunk c start once the epilogue has written it
       LB_ACC_FULL = 4 + 2 * LY_MAX_NB, LB_ACC_EMPTY, LB_WIN_FULL, LB_WIN_EMPTY, LB_H_EMPTY, LB_H_FULL,
       // fused, CTA pairs: the receiver's hidden rows [0, MIR) of its first tile, written and arrived on by the giver's
       // epilogue warps (fz_run)
       LB_H_HALO = LB_H_FULL + LY_H_CHUNKS,
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
  int stage_bytes;             // bytes of one ring stage: b_chunk_bytes (+ 4 * WIN * 16 when the A pair rides along)
  int b_chunk_bytes;           // bytes of one weight chunk, hi and lo: LY_KC * 2 planes of 2 NS (SPLIT) or 2 N columns
  int n_bchunks;               // weight chunks per tile
  int tl_enable;               // timeline builds only: this launch flushes its events
  // one-launch step for stacks with one hidden layer (the FUSED instantiation): t.st[0] is the hidden layer, t.st[1] the
  // heads; both weight images are resident, the hidden activations stay in shared memory
  int sm_h;                    // fused: the hidden operand buffer [chunk][TC_TILE + MIR][8] hi, then lo
  int sm_b1, sm_bias1;         // fused: the heads' resident weights and bias table
  int n_bchunks1, b_chunk_bytes1;
  int paired;                  // fused: launched in clusters of two CTAs that share a halo (fz_run)
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
// the three split products, accumulating in registers (returned in acc[0, 8 SPG) with the correction sum added).  A
// span of contiguous columns of a B image is one K-major descriptor (8-column groups 128 B apart, the two K halves one
// plane apart).  SPLIT stages (NGW <= LY_SPLIT_NGW) hold [W_lo | W_hi] in each K plane, so A_hi is fetched once for both
// of its products: per K-step and tap, the correction sum acc[0, 8 SPG) += A_lo W_hi over the span, then one
// instruction of twice the span computes A_hi [W_lo | W_hi] into all of acc, the main sum in acc[8 SPG, 16 SPG).  Each
// sum adds the same products in the same order as three instructions of the span would.  The correction sum comes
// first because ptxas keeps a wgmma whose accumulators are a prefix of the next one's asynchronous, and serializes
// every wgmma of the kernel when they are a suffix.  Wider stages issue each product as one wgmma over the span (NI = 1),
// or for 160 columns two of half the span (NI = 2): an m64n160 instruction needs more registers than the launch's 96 by
// itself, although all 80 accumulators fit after setmaxnreg.  The halves' fragments sit side by side in acc exactly as
// one instruction's would.  NGW is a compile-time count: a span past the stage's columns computes on zeros (SPLIT) or
// on whatever follows in shared memory -- the next K plane, the next image, or the LY_B_SLACK bytes every layout
// reserves past its last one -- and is not stored, so every wgmma is issued unconditionally and ptxas keeps them
// asynchronous.
//   ring: the tile's weight chunks are the CTA's gchunk, gchunk + 1, ... (every tile streams all n_chunks); chunk g sits
//   in ring stage g % NB (parity from g / NB), released after its MMAs complete;
//   otherwise resident: chunk c sits in stage c behind barrier bar0 + c (parity 0).
//   a_in_stage: the A chunk pair of K-step c rides in the ring stage before the weights; otherwise A is a window at a_addr,
//   and barrier a_release (if >= 0) is arrived on once the MMAs have read it.  a_full (if >= 0): chunk c of the window
//   is written while earlier chunks are multiplied, and its MMAs wait on barrier a_full + c (parity a_parity).
// the two MMA warpgroups converge here before a stage's MMAs: without a barrier between the per-thread mbarrier waits
// and the accumulator set-up, ptxas treats the wgmma sequence as divergent code and serializes every wgmma
__device__ __forceinline__ void mma_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(LY_MMA_WARPS * 32) : "memory"); }
// the epilogue warps alone
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 2, %0;" ::"n"(LY_ETHREADS) : "memory"); }

template <int SPG, bool SPLIT>
__device__ __forceinline__ void ly_mma_tile(float* acc, uint64_t* bars, int N, int col0, int n_chunks, bool ring, int NB,
                                            int gchunk, int bar0, uint32_t b_addr0, uint32_t stage_bytes,
                                            uint32_t b_lo_off, bool a_in_stage, uint32_t a_addr, uint32_t a_plane,
                                            uint32_t a_lo_off, int Wp, int a_release, int a_full = -1,
                                            uint32_t a_parity = 0u) {
  constexpr int NA = 8 * SPG;          // accumulators per thread: 64 x 16 SPG over the 128 threads of the warpgroup
  constexpr int NI = SPG > 8 ? 2 : 1;  // wgmma instructions per product
  constexpr int GI = SPG / NI;         // 16-column groups per instruction
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rh = warp >> 2, wl = warp & 3;
  // bytes per K plane of the B image: SPLIT, the span's lo and hi columns; otherwise the N columns of the hi (lo) image,
  // whose chunk sits b_lo_off bytes after the hi one's in a ring stage
  const uint32_t b_plane = SPLIT ? 2u * 16u * SPG * 16u : (uint32_t)N * 16u;
  const uint32_t sh[IAF_NTAPS] = {0u, 1u, (uint32_t)(Wp - 1), (uint32_t)Wp, (uint32_t)(Wp + 1)};  // 16-byte units
  const uint32_t a_kstep = (2u * a_plane) >> 4, b_tstep = (2u * b_plane) >> 4;
  const uint32_t a_row = (uint32_t)(rh * 64);  // 64 slots = 64 descriptor units
  // The two correction products (lo x hi, hi x lo: 2^-11 of hi x hi) go to their own accumulators where registers allow:
  // added one by one to the main sum, each is rounded at the main sum's magnitude by the tensor cores' accumulation, and
  // over K = 160 those roundings reach ~2e-7 of a unit pre-activation -- enough to put a ReLU's derivative on the wrong
  // side of a pre-activation that small.  Summed apart and added once at the end, they cost one rounding.  Stages of at
  // most 64 columns do so, in acc[0, NA), the main sum in acc[NA, 2 NA).
#pragma unroll
  for (int e = 0; e < (SPLIT ? 2 : 1) * NA; ++e) acc[e] = 0.f;
  int prev_stg = -1;
  for (int c = 0; c < n_chunks; ++c) {
    const int stg = ring ? (int)((uint32_t)gchunk % (uint32_t)NB) : c;
    mbar_wait(&bars[bar0 + stg], ring ? ((uint32_t)gchunk / (uint32_t)NB) & 1u : 0u);
    if (a_full >= 0) mbar_wait(&bars[a_full + c], a_parity);
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
    const uint32_t bl0 = SPLIT ? 0u : wg_desc_lo(bbase + b_lo_off, b_plane) + (uint32_t)col0;
    wgmma_fence();
#pragma unroll 1
    for (int t = 0; t < IAF_NTAPS; ++t) {
      const uint64_t ah = mk_desc(ah0 + sh[t]), al = mk_desc(al0 + sh[t]);
      const uint32_t bt = (uint32_t)t * b_tstep;
      if constexpr (SPLIT) {
        wgmma_m64nNk16<SPG>(acc, al, mk_desc(bh0 + bt + 16u * SPG));  // W_hi: NS columns into the plane
        wgmma_m64nNk16<2 * SPG>(acc, ah, mk_desc(bh0 + bt));
      } else {
#pragma unroll
        for (int h = 0; h < NI; ++h) {  // instruction h: columns [16 GI h, +16 GI), 16 B per column in the descriptor
          const uint32_t bc = bt + (uint32_t)(16 * GI * h);
          wgmma_m64nNk16<GI>(acc + 8 * GI * h, al, mk_desc(bh0 + bc));
          wgmma_m64nNk16<GI>(acc + 8 * GI * h, ah, mk_desc(bl0 + bc));
          wgmma_m64nNk16<GI>(acc + 8 * GI * h, ah, mk_desc(bh0 + bc));
        }
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
    for (int e = 0; e < NA; ++e) acc[e] = acc[NA + e] + acc[e];
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

// The one-launch kernel's run of tiles for CTA b of a grid of G over NT tiles: `n` tiles from `first`, in descending
// order if `desc`, and whether the run's first tile computes its halo rows itself (`halo`) or receives them.
//   unpaired: CTA b runs [floor(b NT / G), floor((b + 1) NT / G)) upwards, each run with a halo block.
//   paired (clusters of two CTAs, G even): cluster c of G / 2 covers [T0, T2) = [floor(c NT / (G / 2)),
//   floor((c + 1) NT / (G / 2))), split at T1 = T0 + floor((T2 - T0) / 2).  Rank 0, the giver, runs [T0, T1) downwards
//   from T1 - 1; rank 1, the receiver, runs [T1, T2) upwards, so the larger half of an odd split goes to the receiver,
//   which then has no halo block on its critical path.  Both first tiles need the hidden rows of slots [TC_TILE T1,
//   +MIR): the giver computes them in its halo block and also writes them into the receiver's buffer.  Where two
//   clusters meet, both runs end and each last tile carries its rows from the tile before it.  A cluster of one tile
//   has an empty lower run, and its receiver runs as an unpaired CTA.
// 32-bit products: NT < 2^24 (tc_num_tiles) and G is at most the SM count.
struct FzRun { int first, n, desc, halo; };
__host__ __device__ inline FzRun fz_run(int b, int G, int NT, bool paired) {
  if (!paired) {
    const int a = (int)((uint32_t)b * (uint32_t)NT / (uint32_t)G), e = (int)((uint32_t)(b + 1) * (uint32_t)NT / (uint32_t)G);
    return FzRun{a, e - a, 0, 1};
  }
  const uint32_t nc = (uint32_t)G / 2u, c = (uint32_t)b / 2u;
  const int T0 = (int)(c * (uint32_t)NT / nc), T2 = (int)((c + 1u) * (uint32_t)NT / nc);
  const int T1 = T0 + (T2 - T0) / 2;
  if (T1 == T0) return (b & 1) ? FzRun{T1, T2 - T1, 0, 1} : FzRun{T0, 0, 0, 0};
  return (b & 1) ? FzRun{T1, T2 - T1, 0, 0} : FzRun{T1 - 1, T1 - T0, 1, 1};
}

// NGW: ceil(N / 32); an MMA warpgroup covers the stage's columns as 2 NGW groups of 16.  Tile t covers slots
// [TC_TILE t, +TC_TILE) in both kernels.  FUSED: the whole step of a one-hidden-layer stack in one launch (NGW covers
// both stages).  Each CTA runs one contiguous run of tiles (fz_run).  Row j of the hidden buffer holds slot
// TC_TILE t + j, j < TC_TILE + MIR, since the heads' taps read up to MIR rows ahead.  Upwards, a tile's hidden MMAs
// compute rows [MIR, TC_TILE + MIR) from a z window that starts MIR slots into the tile; rows [0, MIR) are the previous
// tile's rows [TC_TILE, TC_TILE + MIR), carried to the front once its heads MMAs have released the buffer.  Downwards,
// a tile computes rows [0, TC_TILE) from a window at its first slot, and rows [TC_TILE, TC_TILE + MIR) are the previous
// tile's rows [0, MIR), carried to the back.  The run's first tile gets those rows from a halo block: a hidden pass
// over a z window of its own at the first slot they hold, whose first 64 rows (MIR <= 64, fz_layout) are kept -- or,
// for a pair's receiver, from its giver's halo block.  Both MMA warpgroups issue the same wgmma sequence either way;
// the direction changes only window slots and buffer rows.  A hidden row adds the same products in the same order
// whichever tile computes it.
template <bool PADW, int MODE, int NLT, int NGW, bool FUSED>
__global__ void __launch_bounds__(LY_THREADS, 1) iaf_ly_kernel(const __grid_constant__ IafLyParams q) {
  const IafTcParams& p = q.t;
  const int HW = p.HW;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[LB_COUNT];
  __shared__ int s_win_next[2];  // first stage: the next unclaimed z-window item of the tiles with parity 0 / 1
  TL_DECL

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const IafTcStage& St0 = p.st[0];
  const int nchunk = St0.cin >> 3;
  const int a_plane = p.WIN * 16;          // bytes per chunk plane of the A window
  const int a_lo_off = nchunk * a_plane;
  // tiles of this CTA, i = 0 .. n_my - 1: fused, the run of fz_run from t0, up or (desc) down (which tile covers which
  // slots does not depend on the grid, only which CTA runs it); per stage, u = blockIdx.x + i * gridDim.x.  They live in
  // shared memory and are read where they are used: a register holding them through the whole kernel spilled at the
  // launch's 96
  __shared__ int s_run[4];
  const int& t0 = s_run[0];
  const int& n_my = s_run[1];
  // fused: whether the run goes down, and 1 if it has a halo block, which takes window and accumulator use 0 (per stage,
  // 0 and 0)
  auto desc = [&]() { return FUSED ? s_run[2] : 0; };
  auto W0 = [&]() { return FUSED ? s_run[3] : 0; };
  auto tile_of = [&](int i) { return FUSED ? (desc() ? t0 - i : t0 + i) : (int)blockIdx.x + i * (int)gridDim.x; };
  // z windows, use w: fused, w = 0 the halo block's (if any; at the first slot of the rows it keeps) and w = i + W0
  // tile i's (upwards MIR slots into the tile, downwards at its first slot); per stage, w = i is tile i's
  auto win_slot0 = [&](int w) {
    if (!FUSED) return TC_TILE * tile_of(w);
    return w < W0() ? TC_TILE * (t0 + desc()) : TC_TILE * tile_of(w - W0()) + (desc() ? 0 : p.MIR);
  };
  const bool resident = FUSED || q.n_bchunks <= q.NB;
  const bool ring = !resident || q.in_mode;
  // an MMA warpgroup's span: all 32 NGW columns, or for NGW = 6 two passes over K of 96 columns each (the ring streams
  // the tile's chunks once per pass)
  constexpr int NP = NGW > 5 ? 2 : 1;
  constexpr int SPG = 2 * NGW / NP;
  constexpr bool SPLIT = NGW <= LY_SPLIT_NGW;
  constexpr int REGS_MMA = ly_regs_mma(NGW), REGS_AUX = ly_regs_aux(NGW);

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
      mbar_init(&bars[LB_WIN_FULL], LY_WIN_WARPS + LY_EPI_WARPS);
      s_win_next[0] = s_win_next[1] = 0;
      if (FUSED) {
        const FzRun r = fz_run((int)blockIdx.x, (int)gridDim.x, p.NT, q.paired != 0);
        s_run[0] = r.first; s_run[1] = r.n; s_run[2] = r.desc; s_run[3] = r.halo;
      } else {
        s_run[0] = (int)blockIdx.x;
        s_run[1] = (int)((uint32_t)(p.NT - (int)blockIdx.x + (int)gridDim.x - 1) / gridDim.x);
      }
      mbar_init(&bars[LB_WIN_EMPTY], 2);
      for (int c = 0; c < LY_H_CHUNKS; ++c) mbar_init(&bars[LB_H_FULL + c], LY_EPI_WARPS);
      mbar_init(&bars[LB_H_EMPTY], 2);
      mbar_init(&bars[LB_H_HALO], LY_EPI_WARPS);  // every epilogue warp of the giver arrives
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
  // paired: the barrier also makes each CTA's initialised LB_H_HALO visible to the other before the giver arrives on it
  if (FUSED && q.paired) cluster_sync();
  else __syncthreads();

  // fp32 z (layer mode: post_mean + exp(post_logsd) z) -> the fp16 hi/lo A window of the CTA's w-th use (first stage).
  // Items are (chunk of 8 channels, window slot).  The builder warps and, once their hidden epilogue is done, the
  // epilogue warps claim them 32 K at a time from the use's counter, so the window is shared by whoever is free; each
  // lane keeps the loads of its K items in flight.  Then the warp hands its part to the MMAs.
  auto build_window = [&](int w, auto k_) {
    constexpr int K = decltype(k_)::value;
    const int s0 = win_slot0(w);
    const int n_items = p.WIN * nchunk;
#pragma unroll 1
    for (;;) {
      int base = 0;
      if (lane == 0) base = atomicAdd(&s_win_next[w & 1], 32 * K);
      base = __shfl_sync(0xffffffffu, base, 0);
      if (base >= n_items) break;
      float v[K][8];
#pragma unroll
      for (int h = 0; h < K; ++h) {
        const int idx = base + 32 * h + lane;
        const int ch = fast_div(idx, p.WIN, p.mg_win);
        const SlotInfo si = decode_slot(p, s0 + idx - ch * p.WIN, HW);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[h][e] = 0.f;
        if (si.valid && idx < n_items) {
          const size_t g = ((size_t)si.n * p.C + ch * 8) * HW + si.gp;
#pragma unroll
          for (int e = 0; e < 8; ++e) v[h][e] = __ldg(p.z + g + (size_t)e * HW);
          if (MODE == IAF_MODE_LAYER) {
#pragma unroll
            for (int e = 0; e < 8; ++e)
              v[h][e] = fmaf(fast_exp(__ldg(p.post_logsd + g + (size_t)e * HW)), v[h][e],
                             __ldg(p.post_mean + g + (size_t)e * HW));
          }
        }
      }
#pragma unroll
      for (int h = 0; h < K; ++h) {
        const int idx = base + 32 * h + lane;
        if (idx < n_items) {
          const int ch = fast_div(idx, p.WIN, p.mg_win);
          uint8_t* dst = smem + q.sm_a + ch * a_plane + (idx - ch * p.WIN) * 16;
          split_store8(v[h], dst, dst + a_lo_off);
        }
      }
    }
    fence_proxy_async();  // generic-proxy stores -> the wgmma (async proxy) reads of the window
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[LB_WIN_FULL]);
  };

  if (warp >= LY_TMA_WARP) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS_AUX));
    if (warp == LY_TMA_WARP) {
      // ===================== producer: A windows (operand-image input) and the weight ring =====================
      if (lane == 0 && FUSED) {
        // both stages' weights, resident: hidden chunk c behind barrier c, heads chunk c behind barrier n_bchunks + c
        // (none for an empty run, which must not exit with copies in flight)
        static_assert(!FUSED || SPLIT, "the one-launch kernel's images are [W_lo | W_hi] planes");
        for (int s = 0; s < (n_my > 0 ? 2 : 0); ++s) {
          const IafTcStage& S = p.st[s];
          const int nb = s ? q.n_bchunks1 : q.n_bchunks, bcb = s ? q.b_chunk_bytes1 : q.b_chunk_bytes;
          uint8_t* base = smem + (s ? q.sm_b1 : q.sm_b);
          for (int c = 0; c < nb; ++c) {
            uint64_t* bar = &bars[LB_BFULL + (s ? q.n_bchunks : 0) + c];
            mbar_expect_tx(bar, (uint32_t)bcb);
            bulk_g2s(base + c * bcb, reinterpret_cast<const uint8_t*>(S.whi) + (size_t)c * bcb, (uint32_t)bcb, bar);
          }
        }
      } else if (lane == 0) {
        int gchunk = 0;
        for (int i = 0; i < n_my; ++i) {
          const int u = tile_of(i);
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
            if (q.in_mode) {
              // one ring stage = A chunk pair (hi c0, hi c1, lo c0, lo c1) + the weight chunk of K-step c
              mbar_expect_tx(&bars[LB_BFULL + stg], (uint32_t)(4 * a_plane + q.b_chunk_bytes));
  #pragma unroll
              for (int h = 0; h < 2; ++h) {
                const size_t go = ((size_t)(2 * c + h) * q.S_pad + (size_t)u * TC_TILE) * 8;
                bulk_g2s(dst + h * a_plane, q.a_hi + go, (uint32_t)a_plane, &bars[LB_BFULL + stg]);
                bulk_g2s(dst + (2 + h) * a_plane, q.a_lo + go, (uint32_t)a_plane, &bars[LB_BFULL + stg]);
              }
              dst += 4 * a_plane;
            } else {
              mbar_expect_tx(&bars[LB_BFULL + stg], (uint32_t)q.b_chunk_bytes);
            }
            if (SPLIT) {  // the chunk's planes of the one image
              bulk_g2s(dst, reinterpret_cast<const uint8_t*>(St0.whi) + (size_t)c * q.b_chunk_bytes,
                       (uint32_t)q.b_chunk_bytes, &bars[LB_BFULL + stg]);
            } else {      // the hi half, then the lo half
              const int half = q.b_chunk_bytes / 2;
              const size_t bo = (size_t)c * half;
              bulk_g2s(dst, reinterpret_cast<const uint8_t*>(St0.whi) + bo, (uint32_t)half, &bars[LB_BFULL + stg]);
              bulk_g2s(dst + half, reinterpret_cast<const uint8_t*>(St0.wlo) + bo, (uint32_t)half, &bars[LB_BFULL + stg]);
            }
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
        const int u = tile_of(i);
        const int pb = i & 1;
        const int tile_s0 = u * TC_TILE;
        const int n_first = fast_div(tile_s0, p.SPS, p.mg_sps);
        const int n_last = min(p.B - 1, fast_div(tile_s0 + TC_TILE - 1, p.SPS, p.mg_sps));
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
                const int ta = a / TC_TILE, tbk = bb / TC_TILE;
                const unsigned expected = (unsigned)(tbk - ta + 1);
                __threadfence();
                if (atomicAdd(p.counter + n, 1u) == expected - 1u) {
                  __threadfence();
                  p.counter[n] = 0u;
                  float cost = 0.f;
                  for (int c = 0; c < cred; ++c) {
                    float tot = 0.f;
                    for (int tt = ta; tt <= tbk; ++tt) {
                      const int nf = fast_div(tt * TC_TILE, p.SPS, p.mg_sps);
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
    } else if (warp >= LY_WIN_WARP0 && !q.in_mode) {
      // ===================== window builders: window w once the MMAs have read window w - 1 ================
      // four items per lane in flight at 80 registers, two at 64
      for (int w = 0; w < n_my + W0(); ++w) {
        if (w >= 1) mbar_wait(&bars[LB_WIN_EMPTY], (uint32_t)((w - 1) & 1));
        // every claim on the other counter (window w - 1's) was made before that window was handed over: reset it for
        // window w + 1, whose builders start only after this warp's arrival on window w
        if (warp == LY_WIN_WARP0 && lane == 0) s_win_next[(w + 1) & 1] = 0;
        build_window(w, std::integral_constant<int, (REGS_AUX >= 80 ? 4 : 2)>{});
        if (warp == LY_WIN_WARP0 && lane == 0) TL(3, 10, w);
      }
    }
    // otherwise (operand-image stages, or no per-sample outputs) the warp waits at the closing barrier
  } else if (warp < LY_MMA_WARPS) {
    // ===================== MMA warpgroups: a tile's MMAs run while the epilogue warps finish the previous one =======
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS_MMA));
    float acc[(SPLIT ? 2 : 1) * 8 * SPG];  // SPLIT: room for the correction sum (ly_mma_tile)
    const bool tl0 = warp == 0 && lane == 0;
    if (FUSED && W0()) {
      // the run's halo block: warpgroup 0's hidden rows [0, 64) of window 0 hold the MIR halo rows of the run's first
      // tile.  Warpgroup 1 runs the same K-steps on rows nobody reads: a trip count that differs between the
      // warpgroups makes ptxas serialize every wgmma of the kernel
      mbar_wait(&bars[LB_WIN_FULL], 0u);
      mma_bar_sync();
      ly_mma_tile<SPG, SPLIT>(acc, bars, St0.N, 0, q.n_bchunks, false, 1, 0, LB_BFULL,
                              smem_u32(smem + q.sm_b), (uint32_t)q.b_chunk_bytes, (uint32_t)(q.b_chunk_bytes / 2), false,
                              smem_u32(smem + q.sm_a), (uint32_t)a_plane, (uint32_t)a_lo_off, p.Wp, LB_WIN_EMPTY);
      if (tl0) TL(0, 12, 0);
      ly_acc_store<SPG>(acc, bars, reinterpret_cast<float*>(smem + q.sm_acc), St0.N, 0, 0, true, true);
    }
    for (int i = 0; i < n_my; ++i) {
      if (!q.in_mode) mbar_wait(&bars[LB_WIN_FULL], (uint32_t)((i + W0()) & 1));
      mma_bar_sync();
      if (tl0) TL(0, 15, i);
#pragma unroll 1
      for (int ps = 0; ps < NP; ++ps) {
        if (ps) mma_bar_sync();
        ly_mma_tile<SPG, SPLIT>(acc, bars, St0.N, 16 * SPG * ps, q.n_bchunks, ring, q.NB, (i * NP + ps) * q.n_bchunks,
                                LB_BFULL, smem_u32(smem + q.sm_b), (uint32_t)(FUSED ? q.b_chunk_bytes : q.stage_bytes),
                                (uint32_t)(q.b_chunk_bytes / 2), q.in_mode != 0, smem_u32(smem + q.sm_a), (uint32_t)a_plane,
                                (uint32_t)a_lo_off, p.Wp, (q.in_mode || ps + 1 < NP) ? -1 : (int)LB_WIN_EMPTY);
        if (tl0 && ps + 1 == NP) TL(0, 20, i);
        ly_acc_store<SPG>(acc, bars, reinterpret_cast<float*>(smem + q.sm_acc), St0.N, 16 * SPG * ps,
                          FUSED ? 2 * i + W0() : i, ps == 0, ps + 1 == NP);
      }
      if (tl0) TL(0, 21, i);
      if (FUSED) {
        const IafTcStage& St1 = p.st[1];
        const int h_plane = (TC_TILE + p.MIR) * 16;
        // a pair's receiver: its first tile's rows [0, MIR) come from the giver.  It touches none of them before these
        // MMAs (its hidden epilogue writes rows [MIR, TC_TILE + MIR), the carry waits for these MMAs), so the giver
        // needs no "empty" barrier to write them
        if (!W0() && i == 0) {
          mbar_wait_cluster(&bars[LB_H_HALO], 0u);
          if (tl0) TL(0, 36, i);
        }
        // heads weight chunk c reads hidden channels [16 c, +16): its MMAs start as soon as the epilogue has written
        // them, while it computes the later chunks
        mbar_wait(&bars[LB_H_FULL], (uint32_t)(i & 1));
        mma_bar_sync();
        if (tl0) TL(0, 35, i);
        ly_mma_tile<SPG, SPLIT>(acc, bars, St1.N, 0, q.n_bchunks1, false, 1, 0, LB_BFULL + q.n_bchunks,
                                smem_u32(smem + q.sm_b1), (uint32_t)q.b_chunk_bytes1, (uint32_t)(q.b_chunk_bytes1 / 2),
                                false, smem_u32(smem + q.sm_h), (uint32_t)h_plane, (uint32_t)((St1.cin >> 3) * h_plane),
                                p.Wp, LB_H_EMPTY, LB_H_FULL, (uint32_t)(i & 1));
        if (tl0) TL(0, 40, i);
        ly_acc_store<SPG>(acc, bars, reinterpret_cast<float*>(smem + q.sm_acc), St1.N, 0, 2 * i + 1 + W0(), true,
                          true);
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
    // slot row `row` of the accumulator tile, 8 (16) columns from c0, times the columns' inverse weight scales (exact:
    // powers of two; wsinv null = unscaled images, the data gradient's)
    auto acc_ld8 = [&](int row, int c0, uint32_t* r, int pitch, const float* wsinv) {
      const float4* s4 = reinterpret_cast<const float4*>(s_acc + row * pitch + c0);
#pragma unroll
      for (int e4 = 0; e4 < 2; ++e4) {
        float4 v4 = s4[e4];
        if (wsinv) {
          const float4 w4 = __ldg(reinterpret_cast<const float4*>(wsinv + c0) + e4);
          v4.x *= w4.x; v4.y *= w4.y; v4.z *= w4.z; v4.w *= w4.w;
        }
        r[4 * e4] = __float_as_uint(v4.x); r[4 * e4 + 1] = __float_as_uint(v4.y);
        r[4 * e4 + 2] = __float_as_uint(v4.z); r[4 * e4 + 3] = __float_as_uint(v4.w);
      }
    };
    auto acc_ld16 = [&](int row, int c0, uint32_t* r, int pitch, const float* wsinv) {
      acc_ld8(row, c0, r, pitch, wsinv);
      acc_ld8(row, c0 + 8, r + 8, pitch, wsinv);
    };
    const int h_plane = (TC_TILE + p.MIR) * 16;  // fused: bytes per chunk plane of the hidden operand buffer
    // this warp is done reading the accumulator tile
    auto acc_release = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[LB_ACC_EMPTY]);
    };

    // the epilogue warps' share of window w (which they start once the MMAs have read window w - 1)
    auto help_window = [&](int w) {
      if (w >= 1) mbar_wait(&bars[LB_WIN_EMPTY], (uint32_t)((w - 1) & 1));
      build_window(w, std::integral_constant<int, 2>{});
      if (ew == 0 && lane == 0) TL(1, 10, w);
    };
    if (!q.in_mode && (!FUSED || n_my > 0)) help_window(0);

    for (int i = 0; i < n_my; ++i) {
      const int u = tile_of(i);
      // per stage: help with the next tile's window before this tile's epilogue, which then runs under its MMAs
      if (!FUSED && !q.in_mode && i + 1 < n_my) help_window(i + 1);
      const SlotInfo si_all = decode_slot(p, u * TC_TILE + sl, HW);
      // the accumulator tile's uses: one per tile, or (fused) 0 for the run's halo block if it has one, then 2i + W0 for
      // the hidden stage and 2i + 1 + W0 for the heads.  Each epilogue issues its first input loads (context, z), which
      // do not depend on the MMAs, before waiting on it
      auto acc_wait = [&](uint32_t parity, int tag) {
        mbar_wait(&bars[LB_ACC_FULL], parity);
        if (ew == 0 && lane == 0) TL(1, tag, i);
      };

      // hidden stage epilogue: the next operand (global image, or the fused kernel's shared-memory buffer) for slots
      // TC_TILE u + row0 + [0, TC_TILE).  Warp ew covers slots [32 qd, +32).  Fused: two threads per slot, channels
      // [8 cg, +8) of each 16-channel group, all eight warps on one group at a time, so that the buffer goes to the heads
      // MMAs chunk by chunk, the first after an ngroups-th of the epilogue.  Per stage: one thread per slot and 16
      // channels, groups cg, cg + 2, ...  The halo block's epilogue covers only its first MIR slots, all eight warps
      // over them: warp ew takes slots [32 (ew / HWP), +32) and channels [8 (ew % HWP), +8), every 8 HWP, with HWP = 8
      // warps per 32 slots, or 4 for MIR > 32 -- one 8-channel chunk per thread at c2a, so that its latency is short.
      // Every element is computed the same way under each mapping.  Fused, the rows go to buffer rows [row0, +TC_TILE);
      // the halo block's epilogue hands nothing to its own heads MMAs (tile 0's chunk handoffs cover its rows).  A pair's
      // giver (desc) also writes them to rows [0, MIR) of its receiver's buffer (rank 1 of the cluster, fz_run) and
      // arrives on the receiver's LB_H_HALO.
      constexpr int HC = FUSED ? 8 : 16;  // channels per thread and group
      auto hidden_epi = [&](const IafTcStage& St, const float* tb, const int ngroups, const int pitch,
                            uint32_t acc_parity, const int row0, const bool halo) {
        const int HWP = p.MIR > 32 ? 4 : 8;
        const int sr = halo ? 32 * (ew / HWP) + lane : sl;  // this thread's slot row
        const SlotInfo si = decode_slot(p, u * TC_TILE + row0 + sr, HW);
        const bool bx0 = (si.x == 0), bxW = (si.x == p.W - 1), byH = (si.y == p.H - 1);
        // store_row: the halo block writes MIR buffer rows only (its later rows are the first tile's own).
        // keep_row: every slot's fp32 activations (hid_out) are written once.  The halo block keeps its MIR rows.  Where
        // a tile upwards computes its last MIR rows, the next tile's first, it keeps them only when the next tile is in
        // its run: otherwise they are the first rows of a run that starts there (kept by its halo block, or by its
        // giver's) or of a run that ends there downwards (kept by its last tile, which keeps all its rows)
        const bool store_row = !halo || sr < p.MIR;
        const bool keep_row = halo ? sr < p.MIR : (!FUSED || desc() || sr + p.MIR < TC_TILE || i + 1 < n_my);
        const bool send = FUSED && halo && desc();
        auto store_operand = [&](const float* v8, int chunk) {
          if (FUSED) {
            const int lo = (St.N >> 3) * h_plane;
            uint8_t* dst = smem + q.sm_h + chunk * h_plane + (row0 + sr) * 16;
            if (store_row) {
              uint4 vh, vl;
              split8(v8, vh, vl);
              *reinterpret_cast<uint4*>(dst) = vh;
              *reinterpret_cast<uint4*>(dst + lo) = vl;
              if (send) {
                const uint32_t r = cluster_map(smem + q.sm_h + chunk * h_plane + sr * 16, 1);
                st_cluster16(r, vh);
                st_cluster16(r + lo, vl);
              }
            }
          } else {
            const size_t go = ((size_t)chunk * q.S_pad + (size_t)u * TC_TILE + sr) * 8;
            split_store8(v8, reinterpret_cast<uint8_t*>(q.o_hi + go), reinterpret_cast<uint8_t*>(q.o_lo + go));
          }
        };
          // this thread's HC columns: from c_first, every c_step.  The context of the NEXT ones is fetched while the
          // current ones are computed
          const int nc = 16 * ngroups;
          const int c_first = !FUSED ? 16 * cg : halo ? 8 * (ew % HWP) : 8 * cg;
          const int c_step = !FUSED ? 16 * CGS : halo ? 8 * HWP : 16;
          float cxn[HC];
          auto fetch_ctx = [&](int c0) {
            if (q.first && si.valid && c0 < nc) {  // += context   (ar.py:402 / layers.py:163)
              const float* cp = p.ctx + ((size_t)si.n * St.N + c0) * HW + si.gp;
  #pragma unroll
              for (int e = 0; e < HC; ++e) cxn[e] = __ldg(cp + (size_t)e * HW);
            } else {
  #pragma unroll
              for (int e = 0; e < HC; ++e) cxn[e] = 0.f;
            }
          };
          fetch_ctx(c_first);
          if (FUSED && !halo && i >= 1) {
            // fused: refill the buffer once the heads MMAs of tile i - 1 have read it, first carrying its rows
            // [TC_TILE, TC_TILE + MIR) to the front, or downwards its rows [0, MIR) to the back (every plane), all of
            // them read before any warp overwrites them
            mbar_wait(&bars[LB_H_EMPTY], (uint32_t)((i - 1) & 1));
            const int from = desc() ? 0 : TC_TILE, to = desc() ? TC_TILE : 0;
            for (int k = et; k < 2 * (St.N >> 3) * p.MIR; k += LY_ETHREADS) {
              const int pl = k / p.MIR, rw = k - pl * p.MIR;
              uint4* rows = reinterpret_cast<uint4*>(smem + q.sm_h + pl * h_plane);
              rows[to + rw] = rows[from + rw];
            }
            epi_bar_sync();
            if (ew == 0 && lane == 0) TL(1, 24, i);
          }
          acc_wait(acc_parity, halo ? 13 : 25);
          for (int c0 = c_first; c0 < nc; c0 += c_step) {
            float cx[HC];
  #pragma unroll
            for (int e = 0; e < HC; ++e) cx[e] = cxn[e];
            fetch_ctx(c0 + c_step);
            uint32_t r[HC];
            if (HC == 8) acc_ld8(sr, c0, r, pitch, St.wsinv);
            else acc_ld16(sr, c0, r, pitch, St.wsinv);
            if (q.bwd) {
              // data gradient: acc = (c W)^T g (scaled units); / c (exact: a power of two), x nl'(h), evaluated from the
              // activation itself
              const float sc = si.valid ? dg_scale_from_amax(__ldg(q.amax + si.n)) : 1.0f;
              const float inv = 1.0f / sc;
              const float winv = 1.0f / __ldg(q.wscale);
              float vb[HC];
  #pragma unroll
              for (int e = 0; e < HC; ++e) {
                const float a = __uint_as_float(r[e]) * winv;
                const float d = (q.bwd == 1) ? dg_nl_grad(cx[e], p.nl) : 1.0f;
                vb[e] = si.valid ? a * d : 0.f;
              }
              if (St.hid_out && si.valid && keep_row) {
                float* hp = St.hid_out + ((size_t)si.n * St.N + c0) * HW + si.gp;
                if (q.bwd == 2) {
  #pragma unroll
                  for (int e = 0; e < HC; ++e) hp[(size_t)e * HW] += vb[e] * inv;
                } else {
  #pragma unroll
                  for (int e = 0; e < HC; ++e) hp[(size_t)e * HW] = vb[e] * inv;
                }
              }
              if (q.o_hi) {
  #pragma unroll
                for (int hch = 0; hch < HC / 8; ++hch) store_operand(vb + 8 * hch, (c0 >> 3) + hch);
              }
            } else {
            float v[HC];
            {
              // branch-free: bias rows come in as 16-byte vectors, the pad-channel terms (conv.py:77-83: the pad
              // channel is 1 where a tap falls outside the image) are 0/1-weighted FMAs, and an invalid slot
              // (pad column, zero row, past the end) is selected to zero: that zero IS the conv's padding.  A select, not
              // a multiply: the zero row of sample n - 1 is computed from row 0 of sample n (every tap shift is
              // forward), and NaN * 0 would carry a non-finite sample n into its neighbour's outputs
              const float4* tb4 = reinterpret_cast<const float4*>(tb + c0);
              float bsv[HC];
  #pragma unroll
              for (int e4 = 0; e4 < HC / 4; ++e4) {
                const float4 t4 = tb4[e4];
                bsv[4 * e4] = t4.x; bsv[4 * e4 + 1] = t4.y; bsv[4 * e4 + 2] = t4.z; bsv[4 * e4 + 3] = t4.w;
              }
              if (PADW) {
                const float f1 = bxW ? 1.f : 0.f, f2 = (byH || bx0) ? 1.f : 0.f, f3 = byH ? 1.f : 0.f,
                            f4 = (byH || bxW) ? 1.f : 0.f;
  #pragma unroll
                for (int e = 0; e < HC; ++e)
                  bsv[e] += f1 * tb[St.N + c0 + e] + f2 * tb[2 * St.N + c0 + e] + f3 * tb[3 * St.N + c0 + e] +
                            f4 * tb[4 * St.N + c0 + e];
              }
  #pragma unroll
              for (int e = 0; e < HC; ++e) {
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
            if (St.hid_out && si.valid && keep_row) {  // training forward: keep the activations for iaf_step_bwd_saved
              float* hp = St.hid_out + ((size_t)si.n * St.N + c0) * HW + si.gp;
  #pragma unroll
              for (int e = 0; e < HC; ++e) hp[(size_t)e * HW] = v[e];
            }
  #pragma unroll
            for (int hch = 0; hch < HC / 8; ++hch) store_operand(v + 8 * hch, (c0 >> 3) + hch);
            }
            if (FUSED && !halo) {  // chunk c0 / 16 of the buffer (both of its planes, all slots) goes to the heads MMAs
              fence_proxy_async();  // generic-proxy stores -> the heads' wgmma reads of the buffer
              __syncwarp();
              if (lane == 0) mbar_arrive(&bars[LB_H_FULL + (c0 >> 4)]);
              if (ew == 0 && lane == 0) TL(1, 26 + (c0 >> 4), i);
            }
          }
          if (send) {  // the receiver's rows are written: its heads MMAs (async proxy) may read them
            fence_proxy_async_cluster();
            __syncwarp();
            if (lane == 0) mbar_arrive_cluster(cluster_map(&bars[LB_H_HALO], 1));
            if (ew == 0 && lane == 0) TL(1, 16, i);
          }
      };
      // heads epilogue: affine update, per-element and per-sample outputs
      auto heads_epi = [&](const IafTcStage& St, const float* tb, const int ngroups, const int pitch, const SlotInfo si,
                           uint32_t acc_parity, int acc_tag) {
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
          const bool bx0 = (si.x == 0), bxW = (si.x == p.W - 1), byH = (si.y == p.H - 1);
          const int tile_s0 = u * TC_TILE;
          const int n_first = fast_div(tile_s0, p.SPS, p.mg_sps);
          const int n_last = min(p.B - 1, fast_div(tile_s0 + TC_TILE - 1, p.SPS, p.mg_sps));
          const int ns = (tile_s0 < p.S) ? (n_last - n_first + 1) : 0;
          const int pb = i & 1;
          // z of the NEXT column group is fetched while the current one is computed, the first before the accumulator
          // wait
          float zvn[8];
          auto fetch_z = [&](int g) {
            if (si.valid && g < ngroups) {
              const float* zp = p.z + ((size_t)si.n * p.C + g * 8) * HW + si.gp;
  #pragma unroll
              for (int e = 0; e < 8; ++e) zvn[e] = __ldg(zp + (size_t)e * HW);
            } else {
  #pragma unroll
              for (int e = 0; e < 8; ++e) zvn[e] = 0.f;
            }
          };
          fetch_z(cg);
          if (PERCH && (p.persample_out || p.bc_out) && i >= 2)
            mbar_wait(&bars[LB_PART_EMPTY + pb], (uint32_t)(((i >> 1) - 1) & 1));
          acc_wait(acc_parity, acc_tag);
          for (int g = cg; g < ngroups; g += CGS) {
            const int c0 = g * 16;
            const int ch0 = g * 8;
            float zv[8];
  #pragma unroll
            for (int e = 0; e < 8; ++e) zv[e] = zvn[e];
            fetch_z(g + CGS);
            const size_t gi = si.valid ? ((size_t)si.n * p.C + ch0) * HW + si.gp : 0;
            uint32_t r[16];
            acc_ld16(sl, c0, r, pitch, St.wsinv);
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
        if (i == 0 && W0()) {
          // the first tile's window (once the halo block's MMAs have read theirs) and the halo block's epilogue under
          // the first tile's hidden MMAs: buffer rows [0, MIR) upwards, [TC_TILE, TC_TILE + MIR) downwards.  A giver
          // hands its halo over first, since its receiver's first heads MMAs wait for it
          if (!desc()) help_window(1);
          hidden_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), 0u, desc() ? TC_TILE : 0, true);
          acc_release();
          if (ew == 0 && lane == 0) TL(1, 14, i);
          if (desc()) help_window(1);
        }
        // the hidden epilogue runs under the heads MMAs of its earlier chunks, the heads epilogue under the next tile's
        // hidden MMAs.  Buffer rows [MIR, TC_TILE + MIR) upwards, [0, TC_TILE) downwards
        hidden_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), (uint32_t)W0(), desc() ? 0 : p.MIR, false);
        acc_release();
        if (ew == 0 && lane == 0) TL(1, 30, i);
        // under the heads MMAs: the rest of the next tile's window, beside the builder warps
        if (i + 1 < n_my) help_window(i + 1 + W0());
        const IafTcStage& St1 = p.st[1];
        heads_epi(St1, reinterpret_cast<const float*>(smem + q.sm_bias1), St1.N >> 4, ly_acc_pitch(St1.N), si_all,
                  (uint32_t)(1 - W0()), 45);
        acc_release();
        if (ew == 0 && lane == 0) TL(1, 50, i);
      } else {
        if (!q.is_heads) hidden_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), (uint32_t)(i & 1), 0, false);
        else heads_epi(St0, tb0, St0.N >> 4, ly_acc_pitch(St0.N), si_all, (uint32_t)(i & 1), 25);
        acc_release();
        if (ew == 0 && lane == 0) TL(1, 30, i);
      }
    }
  }

  // paired: neither CTA of the cluster exits while the other may still write to or arrive on its shared memory
  if (FUSED && q.paired) cluster_sync();
  else __syncthreads();
  if (q.tl_enable) {
    if (tid == 0) TL(1, 98, MODE);
    if (tid == 0) TL(1, 99, n_my);
    __syncwarp();
    TL_FLUSH
  }
}
