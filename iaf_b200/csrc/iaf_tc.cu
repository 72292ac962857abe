// Tensor-core path of the IAF step: wgmma implicit GEMM on sm_90a (Hopper).
//
// Formulation.  Every sample's H x W plane is laid out as a stream of "slots" with one
// zero pad column per row and one zero row per sample (pitch Wp = W+1, SPS = (H+1)*Wp
// slots per sample), all samples back to back.  In that stream a conv tap (dy,dx) is a
// pure slot shift of dy*Wp+dx, the SAME zero padding is the pad slots, and every conv
// stage of the masked-AR stack becomes, for every tile of 128 consecutive slots,
//     D[128 x N] = sum over 5 live taps t, channel blocks k:  A_t,k[128 x 16] * W_t,k[16 x N]
// with A_t,k simply the activation matrix read 'shift_t' rows further down.  Activations
// live in shared memory in the wgmma no-swizzle K-major canonical layout
//     [channel chunk of 8][slot][8 x fp16]          (16 B per slot per chunk)
// so a tap shift is +16 B per slot on the descriptor start address.
//
// Precision.  The step must match the fp32 reference to 1e-4 relative; bf16 (or tf32)
// single-pass operands cannot hold that through K = 160..800 and the 8192-element log-det
// sum.  Operands are therefore split x = hi + lo (both fp16, 22 significant bits together;
// see wg_desc_lo) and three MMAs are issued per K block: hi*hi + lo*hi + hi*lo, fp32
// accumulation.  Roofline numbers are always quoted on ALGORITHMIC flops, not on the 3x issued.
//
// Schedule: one launch per conv stage (iaf_tc_gemm.cuh); the same stage kernel runs the data
// gradient of the backward on the point-reflected stream.
// Orientation of the Theano variants: see IafVariantFlags in iaf_common.h (point reflection on load/store, pad-channel
// table; the flipmask variant keeps the table without the reflection).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "iaf_tc.h"

#define TC_TILE 128
#ifdef IAF_TC_TIMELINE
#define TC_SMEM_LIMIT (227 * 1024 - 512 - 9472)  // room for the static event buffers (4 x TL_MAX x 24 B + counts)
#else
#define TC_SMEM_LIMIT (227 * 1024 - 512)  // opt-in maximum minus the kernels' static shared memory (barriers: < 512 B)
#endif
#define TC_ZITEMS 4  // z-window (slot, chunk) items per epilogue thread of the stage kernel

struct IafTcStage {
  const __nv_bfloat16* whi;  // global packed [K/8][N][8]
  const __nv_bfloat16* wlo;
  const float* bias;         // [N] packed column order
  const float* padw;         // [4][N] or nullptr
  const float* wsinv;        // [N] packed column order: the inverse of the power of two each weight column carries
                             // (iaf_tc_pack_kernel), undone as the epilogues read the accumulator tile; nullptr = unscaled
  float* hid_out;            // training forward: this (hidden) stage's activations, fp32 [B][N][HW]; nullptr = not kept
  int cin, N, K;
};

struct IafTcParams {
  const float* z; const float* ctx;
  const float* post_mean; const float* post_logsd; const float* prior_mean; const float* prior_logsd;
  float* z_out; float* elem; float* bc_out; float* persample_out;
  float* logps;              // logp mode: per-element log-density (nullable)
  float* tilepart;           // [NT][MAXS][Cred]
  unsigned* counter;         // [B]
  IafTcStage st[IAF_MAX_STAGES];
  int n_stages;
  int B, C, H, W, Wp, SPS, HW;
  int S;         // total slots
  int NT;        // tiles
  int MIR;       // largest tap shift, rounded up to 8 (slots)
  int WIN;       // A window slots (128 + MIR)
  int MAXS;      // max samples intersecting one tile
  int sm_part;   // smem byte offset of the per-tile partial-sum scratch
  int flip, nl;
  float scale;
  unsigned mg_sps, mg_wp, mg_win;  // magic multipliers for fast_div
};

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// Hopper warpgroup MMA (wgmma), all four warps of a warpgroup converged.  D[64 x 16] += A[64 x 16] * B[16 x 16]: fp16
// operands from shared-memory descriptors (both K-major, or both MN-major with MN = 1), fp32 accumulators in registers.
// Fragment of a thread (warp w of the warpgroup): d[4j + 2h + e] = row 16 w + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e.
template <int MN>
__device__ __forceinline__ void wgmma_m64n16k16(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %11;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a_desc), "l"(b_desc), "r"(1), "n"(MN)
      : "memory");
}
// The same, N = 16 G columns in one instruction (K-major operands): the A tile is fetched once for all N columns
// instead of once per 16.  Fragment: d[4j + 2h + e] = row 16 w + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e, j < 2 G.
// The stage kernel issues G = 2, 4, 5, 6, 8 (see ly_mma_tile).
template <int G>
__device__ __forceinline__ void wgmma_m64nNk16(float* d, uint64_t a_desc, uint64_t b_desc);
template <>
__device__ __forceinline__ void wgmma_m64nNk16<2>(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<4>(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<5>(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<6>(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<8>(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory matrix descriptor, no swizzle, K-major: canonical layout ((8,m),(8,2)):((16B,SBO),(1,LBO)) of
// 8-row x 16-byte core matrices; SBO between 8-row groups (128 B here: rows are linear at 16 B pitch), LBO between the
// two 8-element K chunks of one K = 16 instruction.  Low word: start address >> 4 | (LBO >> 4) << 16.  High word:
// SBO >> 4 (base offset 0, layout type 0 = no swizzle).  Adding n to the low word moves the start by n x 16 bytes.
// Why fp16 pairs and not bf16 pairs: the residual of a two-term WEIGHT split is the same for every pixel and so adds
// up coherently over the 8192 elements of a sample's log-det (bf16 + bf16 leaves 2^-17 |w|, ~2e-4 absolute against the
// fp64 oracle over 256 samples; fp16 + fp16 leaves 2^-23 |w|).  That holds only while the lo half is a normal fp16
// number: below |w| ~ 2^-3 it is subnormal, with a fixed absolute step of 2^-24, so iaf_tc_pack_kernel scales every
// weight column by the power of two that brings its largest |w| into [32, 64) (also keeping gains far above e^11 inside
// the fp16 range) and the stage epilogues divide it out exactly.  See split_store8 for the activations' range.
__device__ __forceinline__ uint32_t wg_desc_lo(uint32_t saddr, uint32_t lbo_bytes) {
  return ((saddr >> 4) & 0x3FFFu) | (((lbo_bytes >> 4) & 0x3FFFu) << 16);
}
#define WG_DESC_HI (128u >> 4)
__device__ __forceinline__ uint64_t mk_desc(uint32_t lo) { return ((uint64_t)WG_DESC_HI << 32) | lo; }

// exp via ex2.approx.ftz (2 ulp): used where 1e-7-level error is far inside the 1e-4 parity budget
__device__ __forceinline__ float fast_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}

// floor(s / d) for 0 <= s < 2^31 with magic = floor(2^32 / d) + 1 (d >= 2): one mul-hi and a fix-up
__device__ __forceinline__ int fast_div(int s, int d, unsigned magic) {
  int q = (int)__umulhi((unsigned)s, magic);
  if (s - q * d < 0) --q;
  return q;
}

template <int NLT>
__device__ __forceinline__ float tc_apply_nl(float v, int nl) {
  if (NLT == IAF_NL_ELU) return v < 0.f ? fast_exp(v) - 1.0f : v;  // abs error ~1e-7, far inside the 1e-4 budget
  switch (nl) {
    case IAF_NL_ELU: return v < 0.f ? fast_exp(v) - 1.0f : v;
    case IAF_NL_SOFTPLUS: return v > 0.f ? v + log1pf(expf(-v)) : log1pf(expf(v));
    case IAF_NL_RELU: return v >= 0.f ? v : 0.f;
    case IAF_NL_TANH: return tanhf(v);
    case IAF_NL_LEAKYRELU: return v < 0.f ? 0.01f * v : v;
    default: return v;
  }
}

// split 8 floats into fp16 hi / lo (22 significant bits together) and store both 16-byte vectors.  fp16, not bf16: the
// a_lo * w_lo product the three-MMA scheme drops and the residual of the two-term split both shrink 64x (CPU simulation
// tools/experiments/prec_sim.py: worst per-sample log-det error on C2a 1.3e-4 with bf16 pairs, 5e-6 with fp16 pairs).
// Range: |x| >= 65520 becomes inf and that sample's outputs NaN (loud, never silently wrong; invalid slots are zeroed by
// a select, so the NaN stays inside its sample).  Activations are not scaled: below |x| ~ 2^-3 the lo half is subnormal
// and x keeps an absolute resolution of about 2^-25 (3e-8) instead of 22 significant bits.
__device__ __forceinline__ void split_store8(const float* v, uint8_t* hi_ptr, uint8_t* lo_ptr) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 hh = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    const float2 hf = __half22float2(hh);
    const __half2 ll = __floats2half2_rn(v[2 * i] - hf.x, v[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hh);
    l[i] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  *reinterpret_cast<uint4*>(hi_ptr) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo_ptr) = make_uint4(l[0], l[1], l[2], l[3]);
}

// Optional in-kernel timeline (compile with -DIAF_TC_TIMELINE; development aid only, tools/tl_run.py): CTA 0 of the
// launch that sets tl_enable records (tag, tile or chunk, clock) triples per role, each at the end of a phase of its own
// warp (other warps of the role may still be in it).  Role 0, lane 0 of MMA warp 0: 15 / 35 the (hidden) / heads MMAs'
// operands ready, 20 / 40 their MMAs done, 21 / 41 their fragments in the accumulator tile (after waiting for the
// epilogues to free it).  Role 1, lane 0 of epilogue warp 0: 10 z window built, 25 / 45 (hidden) / heads accumulators
// ready, 30 (hidden) epilogue done, 50 heads epilogue done (fused), 98 the launch's mode (k = IAF_MODE_*: multiconv,
// step, layer, logp), 99 kernel end.  Role 2, the producer: 60 / 61 before
// / after waiting for a ring stage to be released (k = the weight chunk it will refill).
#ifdef IAF_TC_TIMELINE
#define TL_MAX 96
__device__ long long g_tl[4][TL_MAX][3];
__device__ int g_tl_n[4];
// events are staged in shared memory (a global counter would cost an L2 round trip per event)
#define TL_DECL __shared__ long long s_tl[4][TL_MAX][3]; __shared__ int s_tl_n[4]; if (threadIdx.x < 4) s_tl_n[threadIdx.x] = 0;
#define TL(role, tag, kk)                                                          \
  do {                                                                             \
    if (blockIdx.x == 0) {                                                         \
      const int i_ = s_tl_n[role];                                                 \
      if (i_ < TL_MAX) { s_tl[role][i_][0] = (tag); s_tl[role][i_][1] = (kk); s_tl[role][i_][2] = clock64(); s_tl_n[role] = i_ + 1; } \
    }                                                                              \
  } while (0)
#define TL_FLUSH                                                                   \
  if (blockIdx.x == 0 && threadIdx.x < 4) {                                        \
    const int r_ = threadIdx.x;                                                    \
    for (int i_ = 0; i_ < s_tl_n[r_]; ++i_)                                        \
      for (int c_ = 0; c_ < 3; ++c_) g_tl[r_][i_][c_] = s_tl[r_][i_][c_];          \
    g_tl_n[r_] = s_tl_n[r_];                                                       \
  }
#else
#define TL_DECL
#define TL_FLUSH
#define TL(role, tag, kk) do { } while (0)
#endif

struct SlotInfo {
  int n, y, x, gp;
  bool valid;
};
__device__ __forceinline__ SlotInfo decode_slot(const IafTcParams& p, int s, int HW) {
  SlotInfo si;
  si.n = fast_div(s, p.SPS, p.mg_sps);
  const int r = s - si.n * p.SPS;
  si.y = fast_div(r, p.Wp, p.mg_wp);
  si.x = r - si.y * p.Wp;
  si.valid = (s < p.S) && (si.y < p.H) && (si.x < p.W);
  const int pix = si.y * p.W + si.x;
  si.gp = p.flip ? HW - 1 - pix : pix;
  return si;
}

#include "iaf_tc_gemm.cuh"
#include "iaf_wg.cuh"

// ------------------------------------------------------------------------------------------
// weight preparation for this path: same math as iaf_pack.cu, fp16 hi/lo split, written as
// the wgmma B-operand image [K/8][N][8] (K index [ci / 16][tap][ci % 16], K-major, no swizzle).
// ------------------------------------------------------------------------------------------
struct TcPackLayer {
  const float* w; const float* scale; const float* bias;
  __nv_bfloat16* whi; __nv_bfloat16* wlo; float* bias_out; float* padw_out; float* wsinv_out;
  int cin, cout, N, zerodiag, head, is_head;
};
struct TcPackParams {
  TcPackLayer layer[IAF_MAX_HIDDEN + IAF_MAX_HEADS];
  int n_layers;
  IafVariantFlags vf;
};

// raw weight of canonical tap t, input channel ci (ci == cin: pad channel), output channel co; 0 where not live
__device__ __forceinline__ float tc_masked_weight(const TcPackLayer& L, const IafVariantFlags& vf, int t, int ci, int co) {
  const IafTap tp = iaf_tap_rule(t, ci, co, L.cin, L.cout, L.zerodiag, vf.flipmask);
  return tp.live ? L.w[iaf_raw_index(vf.theano, tp.k, ci, co, L.cin, L.cout)] : 0.f;
}

__global__ void __launch_bounds__(128) iaf_tc_pack_kernel(const __grid_constant__ TcPackParams p) {
  const TcPackLayer& L = p.layer[blockIdx.y];
  const int co = blockIdx.x;
  if (co >= L.cout) return;
  const int tid = threadIdx.x;
  const int n_real = L.cin * IAF_NTAPS;
  // pad channel: taps 1..4; flipped, also its centre, which only enters the norm (see iaf_tap_rule)
  const int n_pad = p.vf.pad_channel ? (p.vf.flipmask ? 5 : 4) : 0;
  const int t_pad0 = IAF_NTAPS - n_pad;
  float ss = 0.f, am = 0.f;  // sum of squares (normalisation, pad channel included) and max |w| of the column's real taps
  for (int e = tid; e < n_real + n_pad; e += blockDim.x) {
    float v;
    if (e < n_real) {
      const int t = e / L.cin, ci = e % L.cin;
      v = tc_masked_weight(L, p.vf, t, ci, co);
      am = fmaxf(am, fabsf(v));
    } else {
      v = tc_masked_weight(L, p.vf, t_pad0 + e - n_real, L.cin, co);
    }
    ss = fmaf(v, v, ss);
  }
  __shared__ float red[128], redm[128];
  red[tid] = ss;
  redm[tid] = am;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (tid < s) {
      red[tid] += red[tid + s];
      redm[tid] = fmaxf(redm[tid], redm[tid + s]);
    }
    __syncthreads();
  }
  ss = red[0];
  const float factor = !p.vf.theano ? expf(L.scale[co]) / sqrtf(fmaxf(ss, 1e-12f))
                                    : expf(3.0f * L.scale[co]) / (sqrtf(ss) + 1e-8f);
  // the column's weight scale: its largest |w| into [32, 64), so that the lo half of every sizeable weight is a normal
  // fp16 number and the largest stays inside the fp16 range.  fl(|v| factor) is monotone in |v|: redm[0] * factor is
  // exactly the largest |v * factor| of the loop below.  The bias and the pad-channel terms stay unscaled fp32.
  const float wsc = dg_scale_from_amax(redm[0] * factor);
  // heads are interleaved in groups of 8: column = (c/8)*16 + head*8 + c%8
  const int col = L.is_head ? ((co >> 3) * 16 + L.head * 8 + (co & 7)) : co;
  for (int e = tid; e < n_real + n_pad; e += blockDim.x) {
    if (e < n_real) {
      const int t = e / L.cin, ci = e % L.cin;
      const float v = tc_masked_weight(L, p.vf, t, ci, co);
      const float vc = v * factor * wsc;  // (a power of two: exact)
      // K order [ci / 16][tap][ci % 16]: one K-step of the stage kernel is one 16-channel block over the five taps
      const int k = ((ci >> 4) * IAF_NTAPS + t) * 16 + (ci & 15);
      // fp16 hi + fp16 lo (22 significant bits)
      const __half hh = __float2half_rn(vc);
      const __half lh = __float2half_rn(vc - __half2float(hh));
      const __nv_bfloat16 h = __ushort_as_bfloat16(__half_as_ushort(hh));  // raw 16-bit patterns travel in the bf16-typed images
      const __nv_bfloat16 l = __ushort_as_bfloat16(__half_as_ushort(lh));
      const size_t o = ((size_t)(k >> 3) * L.N + col) * 8 + (k & 7);  // hi / lo images [K/8][N][8]
      L.whi[o] = h;
      L.wlo[o] = l;
    } else {
      const int t = t_pad0 + e - n_real;
      if (t > 0) L.padw_out[(size_t)(t - 1) * L.N + col] = tc_masked_weight(L, p.vf, t, L.cin, co) * factor;
    }
  }
  if (tid == 0) {
    L.bias_out[col] = L.bias[co];
    L.wsinv_out[col] = 1.0f / wsc;
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
struct IafTcPlan {
  iaf_desc_t d;
  IafVariantFlags vf;
  int n_stages;
  int cin[IAF_MAX_STAGES], N[IAF_MAX_STAGES], K[IAF_MAX_STAGES];
  __nv_bfloat16* whi[IAF_MAX_STAGES];
  __nv_bfloat16* wlo[IAF_MAX_STAGES];
  float* bias[IAF_MAX_STAGES];
  float* padw[IAF_MAX_STAGES];
  float* wsinv[IAF_MAX_STAGES];  // [N]: inverse weight scale of each packed column
  int MIR, WIN, MAXS;
  bool layer_ok;             // the per-(sample,channel) scratch of the fused-layer mode fits
  // one launch per stage: an A window (first stage), an NB-deep ring, the bias table, the partials, the accumulator tile
  int ly_stage[IAF_MAX_STAGES];
  int ly_NB[IAF_MAX_STAGES], ly_sm_a[IAF_MAX_STAGES], ly_sm_b[IAF_MAX_STAGES], ly_sm_bias[IAF_MAX_STAGES],
      ly_sm_part[IAF_MAX_STAGES], ly_sm_acc[IAF_MAX_STAGES];
  size_t ly_smem[IAF_MAX_STAGES];
  // one-launch step (one hidden layer): resident weights of both stages, hidden activations in shared memory
  bool fused;
  int fz_sm_a, fz_sm_h, fz_sm_bias[2], fz_sm_part, fz_sm_acc, fz_sm_b[2];
  size_t fz_smem;
  __nv_bfloat16* img[2][2];  // ping-pong operand images: [which][hi|lo]
  int img_S_pad;
  unsigned* counter;
  float* tilepart;
  int scratch_B, scratch_NT;
  int num_sms;
};

typedef void (*LyKernel)(const IafLyParams);
template <int NGW, bool FUSED>
static LyKernel ly_kernel_pick(bool padw, int mode, bool elu) {
#define LY_PICK(MD)                                                                                                   \
  if (padw) return elu ? iaf_ly_kernel<true, MD, IAF_NL_ELU, NGW, FUSED> : iaf_ly_kernel<true, MD, -1, NGW, FUSED>; \
  return elu ? iaf_ly_kernel<false, MD, IAF_NL_ELU, NGW, FUSED> : iaf_ly_kernel<false, MD, -1, NGW, FUSED>;
  if (mode == IAF_MODE_MULTICONV) { LY_PICK(IAF_MODE_MULTICONV) }
  if (mode == IAF_MODE_STEP) { LY_PICK(IAF_MODE_STEP) }
  if (mode == IAF_MODE_LAYER) { LY_PICK(IAF_MODE_LAYER) }
  LY_PICK(IAF_MODE_LOGP)
#undef LY_PICK
}
// the stage kernel for a stage of N output columns: NGW = ceil(N / 32), an MMA warpgroup's span of 32 NGW columns.  NGW <= 6 (N <=
// 192): wider stages never fit, their accumulator tile [128][N + 4] leaves no room for two ring stages (ly_layout and
// iaf_dg_plan_create reject them before asking for a kernel)
#define LY_MAX_NGW 6
static LyKernel ly_kernel_for(bool padw, int mode, bool elu, int N) {
  switch ((N + 31) / 32) {
    case 1: return ly_kernel_pick<1, false>(padw, mode, elu);
    case 2: return ly_kernel_pick<2, false>(padw, mode, elu);
    case 3: return ly_kernel_pick<3, false>(padw, mode, elu);
    case 4: return ly_kernel_pick<4, false>(padw, mode, elu);
    case 5: return ly_kernel_pick<5, false>(padw, mode, elu);
    default: return ly_kernel_pick<LY_MAX_NGW, false>(padw, mode, elu);
  }
}
// the one-launch step of a one-hidden-layer stack (hidden and 2 n_z at most 64 columns: one m64n64 span)
#define FZ_NGW 2
static LyKernel fz_kernel_for(bool padw, int mode, bool elu) { return ly_kernel_pick<FZ_NGW, true>(padw, mode, elu); }

static int tc_round_up(int a, int b) { return (a + b - 1) / b * b; }

// per stage: an A window (first stage), the bias table, the partial scratch, the accumulator tile, an NB-deep ring.
// A stack without hidden layers (the linear IAF) is one stage, the heads, whose A window is built from fp32 z.
static bool ly_layout(const iaf_desc_t* d, IafTcPlan* pl) {
  if (d->n_heads != 2 || d->head[0] != d->n_z || d->head[1] != d->n_z) return false;
  if (d->n_z % 16 != 0 || 2 * d->n_z > 32 * LY_MAX_NGW) return false;
  for (int i = 0; i < d->n_hidden; ++i)
    if (d->hidden[i] % 16 != 0 || d->hidden[i] > 32 * LY_MAX_NGW) return false;
  const int nst = d->n_hidden + 1;
  const int Wp = d->W + 1;
  const int SPS = (d->H + 1) * Wp;
  const int MIR = tc_round_up(Wp + 1, 8);
  if (MIR > TC_TILE) return false;
  IafTcPlan tmp;
  IafTcPlan* q = pl ? pl : &tmp;
  q->n_stages = nst;
  q->MIR = MIR; q->WIN = TC_TILE + MIR;
  q->MAXS = (TC_TILE - 1) / SPS + 2;
  if ((d->n_z / 8) * q->WIN > TC_ZITEMS * LY_ETHREADS) return false;
  int prev = d->n_z;
  q->layer_ok = true;
  for (int j = 0; j < nst; ++j) {
    q->cin[j] = prev;
    q->N[j] = (j < d->n_hidden) ? d->hidden[j] : 2 * d->n_z;
    q->K[j] = IAF_NTAPS * prev;
    prev = q->N[j];
    int off = 0;
    // first stage: the workers build the whole A window from fp32 z; later stages stream A chunk pairs with the weights
    q->ly_sm_a[j] = off; if (j == 0) off += 2 * (q->cin[j] / 8) * q->WIN * 16;
    q->ly_sm_bias[j] = off; off += 5 * q->N[j] * 4;
    off = tc_round_up(off, 16);
    q->ly_sm_part[j] = off;
    off += std::max(2 * LY_PART_SETS * q->MAXS * 4, 2 * 4 * q->MAXS * d->n_z * 4);
    off = tc_round_up(off, 16);
    q->ly_sm_acc[j] = off; off += TC_TILE * ly_acc_pitch(q->N[j]) * 4;
    off = tc_round_up(off, 128);
    q->ly_sm_b[j] = off;
    const int slot = 2 * LY_KC * 2 * q->N[j] * 16 + (j ? 4 * q->WIN * 16 : 0);  // weight chunk hi+lo (+ A chunk pair hi+lo)
    q->ly_stage[j] = slot;
    int nb = (TC_SMEM_LIMIT - LY_B_SLACK - off) / slot;
    if (nb < 2) return false;
    q->ly_NB[j] = std::min(nb, LY_MAX_NB);
    q->ly_smem[j] = (size_t)off + (size_t)q->ly_NB[j] * slot + LY_B_SLACK;
  }
  return true;
}

// one-launch layout (after ly_layout filled cin / N / K / MIR / WIN / MAXS): A window, hidden operand buffer (TC_TILE + MIR
// rows: the heads' shifted windows of the rows past TS read beyond the 128 computed rows; those rows are not stored), both
// bias tables, the partials, the accumulator tile and both resident weight images
static bool fz_layout(const iaf_desc_t* d, IafTcPlan* q) {
  if (d->n_hidden != 1 || q->N[0] > 32 * FZ_NGW || q->N[1] > 32 * FZ_NGW) return false;
  if (TC_TILE - q->MIR < TC_TILE / 2) return false;
  const int nb0 = q->K[0] / 16 / LY_KC, nb1 = q->K[1] / 16 / LY_KC;
  if (nb0 + nb1 > LY_MAX_NB) return false;
  int off = 0;
  q->fz_sm_a = off; off += 2 * (q->cin[0] / 8) * q->WIN * 16;
  q->fz_sm_h = off; off += 2 * (q->N[0] / 8) * (TC_TILE + q->MIR) * 16;
  for (int j = 0; j < 2; ++j) { q->fz_sm_bias[j] = off; off += 5 * q->N[j] * 4; }
  off = tc_round_up(off, 16);
  q->fz_sm_part = off; off += std::max(2 * LY_PART_SETS * q->MAXS * 4, 2 * 4 * q->MAXS * d->n_z * 4);
  off = tc_round_up(off, 16);
  q->fz_sm_acc = off; off += TC_TILE * ly_acc_pitch(std::max(q->N[0], q->N[1])) * 4;
  off = tc_round_up(off, 128);
  for (int j = 0; j < 2; ++j) { q->fz_sm_b[j] = off; off += 2 * q->K[j] * q->N[j] * 2; }
  off += LY_B_SLACK;
  q->fz_smem = (size_t)off;
  return off <= TC_SMEM_LIMIT;
}

bool iaf_tc_supported(const iaf_desc_t* d) { return ly_layout(d, nullptr); }

int iaf_tc_plan_create(IafTcPlan** out, const iaf_desc_t* d) {
  IafTcPlan* pl = new (std::nothrow) IafTcPlan();
  if (!pl) return IAF_ERR_BAD_ARG;
  memset(pl, 0, sizeof(*pl));
  pl->d = *d;
  pl->vf = iaf_variant_flags(d->variant);
  if (!ly_layout(d, pl)) { delete pl; return IAF_ERR_UNSUPPORTED; }
  // IAF_TC_FUSED=0 (development): one-hidden-layer stacks on the per-stage kernel too, for A/B against the fused one
  const char* fe = getenv("IAF_TC_FUSED");
  pl->fused = !(fe && fe[0] == '0') && fz_layout(d, pl);
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { delete pl; return IAF_ERR_CUDA; }
  if (prop.major != 9) { delete pl; return IAF_ERR_UNSUPPORTED; }  // wgmma: sm_90a
  pl->num_sms = iaf_plan_num_sms(prop.multiProcessorCount);
  for (int j = 0; j < pl->n_stages; ++j) {
    const size_t wb = (size_t)pl->K[j] * pl->N[j] * 2;
    // bias [N] and pad-channel weights [4][N] are ONE table [5][N]; the inverse weight scales [N] follow it
    if (cudaMalloc(&pl->whi[j], wb) != cudaSuccess || cudaMalloc(&pl->wlo[j], wb) != cudaSuccess ||
        cudaMalloc(&pl->bias[j], sizeof(float) * 6 * pl->N[j]) != cudaSuccess) {
      iaf_tc_plan_destroy(pl);
      return IAF_ERR_CUDA;
    }
    pl->padw[j] = pl->bias[j] + pl->N[j];
    pl->wsinv[j] = pl->bias[j] + 5 * pl->N[j];
  }
  for (int a = 0; a < 16; ++a) {
    const int md = a >> 2;  // IAF_MODE_MULTICONV .. IAF_MODE_LOGP
    cudaError_t e = cudaSuccess;
    if (pl->fused) e = iaf_smem_optin(fz_kernel_for(a & 1, md, a & 2));
    for (int j = 0; j < pl->n_stages && e == cudaSuccess && !pl->fused; ++j) e = iaf_smem_optin(ly_kernel_for(a & 1, md, a & 2, pl->N[j]));
    if (e != cudaSuccess) {
      iaf_tc_plan_destroy(pl);
      return IAF_ERR_CUDA;
    }
  }
  *out = pl;
  return IAF_OK;
}

void iaf_tc_plan_destroy(IafTcPlan* pl) {
  if (!pl) return;
  for (int j = 0; j < IAF_MAX_STAGES; ++j) {
    if (pl->whi[j]) cudaFree(pl->whi[j]);
    if (pl->wlo[j]) cudaFree(pl->wlo[j]);
    if (pl->bias[j]) cudaFree(pl->bias[j]);  // padw[j] and wsinv[j] point into the same allocation
  }
  if (pl->counter) cudaFree(pl->counter);
  if (pl->tilepart) cudaFree(pl->tilepart);
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b)
      if (pl->img[a][b]) cudaFree(pl->img[a][b]);
  delete pl;
}
int iaf_tc_pack(IafTcPlan* pl, const float* const* w, const float* const* scale, const float* const* bias,
                cudaStream_t stream) {
  const iaf_desc_t& d = pl->d;
  TcPackParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.n_layers = d.n_hidden + d.n_heads;
  pp.vf = pl->vf;
  int max_cout = 0;
  for (int j = 0; j < pl->n_stages; ++j) {
    const size_t wb = (size_t)pl->K[j] * pl->N[j] * 2;
    if (cudaMemsetAsync(pl->whi[j], 0, wb, stream) != cudaSuccess) return IAF_ERR_CUDA;
    if (cudaMemsetAsync(pl->wlo[j], 0, wb, stream) != cudaSuccess) return IAF_ERR_CUDA;
    if (cudaMemsetAsync(pl->padw[j], 0, sizeof(float) * 4 * pl->N[j], stream) != cudaSuccess) return IAF_ERR_CUDA;
  }
  for (int i = 0; i < pp.n_layers; ++i) {
    TcPackLayer& L = pp.layer[i];
    const bool is_head = i >= d.n_hidden;
    const int j = is_head ? d.n_hidden : i;
    L.w = w[i]; L.scale = scale[i]; L.bias = bias[i];
    L.whi = pl->whi[j]; L.wlo = pl->wlo[j]; L.bias_out = pl->bias[j]; L.padw_out = pl->padw[j];
    L.wsinv_out = pl->wsinv[j];
    L.cin = pl->cin[j];
    L.cout = is_head ? d.head[i - d.n_hidden] : d.hidden[i];
    L.N = pl->N[j];
    L.zerodiag = is_head ? 1 : 0;
    L.is_head = is_head ? 1 : 0;
    L.head = is_head ? i - d.n_hidden : 0;
    max_cout = std::max(max_cout, L.cout);
  }
  dim3 grid(max_cout, pp.n_layers);
  iaf_tc_pack_kernel<<<grid, 128, 0, stream>>>(pp);
  return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
}

#ifdef IAF_TC_TIMELINE
extern "C" void iaf_tc_timeline_dump(void) {
  cudaDeviceSynchronize();
  static long long h[4][TL_MAX][3];
  int n[4];
  cudaMemcpyFromSymbol(h, g_tl, sizeof(h));
  cudaMemcpyFromSymbol(n, g_tl_n, sizeof(n));
  long long t0 = -1;
  for (int r = 0; r < 4; ++r)
    for (int i = 0; i < n[r] && i < TL_MAX; ++i)
      if (t0 < 0 || h[r][i][2] < t0) t0 = h[r][i][2];
  for (int r = 0; r < 4; ++r)
    for (int i = 0; i < n[r] && i < TL_MAX; ++i)
      printf("TL role=%d tag=%lld k=%lld t=%lld\n", r, h[r][i][0], h[r][i][1], h[r][i][2] - t0);
  int z[4] = {0, 0, 0, 0};
  cudaMemcpyToSymbol(g_tl_n, z, sizeof(z));
}
#endif

bool iaf_tc_mode_supported(const IafTcPlan* pl, int mode) {
  // the logp mode shares the layer mode's per-(sample, channel) partials and scratch, so it is available exactly where
  // the layer mode is
  return mode == IAF_MODE_STEP || mode == IAF_MODE_MULTICONV ||
         ((mode == IAF_MODE_LAYER || mode == IAF_MODE_LOGP) && pl->layer_ok);
}

// tiles of a call at batch B (0: the slot stream overflows int)
static int tc_num_tiles(const IafTcPlan* pl, int B) {
  const int SPS = (pl->d.H + 1) * (pl->d.W + 1);
  if ((long long)B * SPS + TC_TILE >= (1LL << 31)) return 0;
  const int TS = pl->fused ? TC_TILE - pl->MIR : TC_TILE;  // slots a tile advances (fused: overlapped windows)
  return (B * SPS + TS - 1) / TS;
}

int iaf_tc_scratch_need(const IafTcPlan* pl, int B) {
  const int NT = tc_num_tiles(pl, B);
  if (NT == 0 || (B <= pl->scratch_B && NT <= pl->scratch_NT)) return IAF_SCRATCH_FITS;  // (overflow: refused, no growth)
  return pl->scratch_B > 0 ? IAF_SCRATCH_REALLOC : IAF_SCRATCH_ALLOC;
}

int iaf_tc_run(IafTcPlan* pl, const IafTcArgs* a, cudaStream_t stream, int* n_launches) {
  const iaf_desc_t& d = pl->d;
  const int B = a->B;
  const int SPS = (d.H + 1) * (d.W + 1);
  const int NT = tc_num_tiles(pl, B);
  if (NT == 0) return IAF_ERR_UNSUPPORTED;
  const int S = B * SPS;
  const int TS = pl->fused ? TC_TILE - pl->MIR : TC_TILE;
  if (B > pl->scratch_B || NT > pl->scratch_NT) {
    if (pl->counter) cudaFree(pl->counter);
    if (pl->tilepart) cudaFree(pl->tilepart);
    pl->counter = nullptr; pl->tilepart = nullptr; pl->scratch_B = 0;
    int maxc = 0;
    for (int j = 0; j + 1 < pl->n_stages; ++j) maxc = std::max(maxc, pl->N[j]);
    pl->img_S_pad = (NT + 1) * TC_TILE;  // one zero tile past the end: windows of the last tile read into it
    const size_t bytes = (size_t)(maxc / 8) * pl->img_S_pad * 16;
    for (int a2 = 0; a2 < 2; ++a2)
      for (int b2 = 0; b2 < 2; ++b2) {
        if (pl->img[a2][b2]) cudaFree(pl->img[a2][b2]);
        pl->img[a2][b2] = nullptr;
        if (maxc == 0) continue;  // no hidden stage: no operand images
        if (cudaMalloc(&pl->img[a2][b2], bytes) != cudaSuccess) return IAF_ERR_CUDA;
        if (cudaMemsetAsync(pl->img[a2][b2], 0, bytes, stream) != cudaSuccess) return IAF_ERR_CUDA;
      }
    if (cudaMalloc(&pl->counter, sizeof(unsigned) * (size_t)B) != cudaSuccess) return IAF_ERR_CUDA;
    if (cudaMemsetAsync(pl->counter, 0, sizeof(unsigned) * (size_t)B, stream) != cudaSuccess) return IAF_ERR_CUDA;
    if (cudaMalloc(&pl->tilepart, sizeof(float) * (size_t)NT * pl->MAXS * d.n_z) != cudaSuccess) return IAF_ERR_CUDA;
    pl->scratch_B = B;
    pl->scratch_NT = NT;
  }
  IafTcParams p;
  memset(&p, 0, sizeof(p));
  p.z = a->z; p.ctx = a->ctx; p.post_mean = a->post_mean; p.post_logsd = a->post_logsd;
  p.prior_mean = a->prior_mean; p.prior_logsd = a->prior_logsd;
  p.z_out = a->z_out;
  p.elem = a->elem_out;
  p.bc_out = a->bc_out; p.persample_out = a->persample_out;
  p.logps = a->logps_out;
  p.tilepart = pl->tilepart;
  p.counter = pl->counter;
  p.n_stages = 1;
  p.B = B; p.C = d.n_z; p.H = d.H; p.W = d.W; p.Wp = d.W + 1; p.SPS = SPS; p.HW = d.H * d.W;
  p.S = S; p.NT = NT;
  p.MIR = pl->MIR; p.WIN = pl->WIN; p.MAXS = pl->MAXS;
  p.flip = pl->vf.reflect;
  p.nl = d.nl; p.scale = 0.1f;
  p.mg_sps = (unsigned)((1ULL << 32) / (unsigned)SPS) + 1u;
  p.mg_wp = (unsigned)((1ULL << 32) / (unsigned)p.Wp) + 1u;
  p.mg_win = (unsigned)((1ULL << 32) / (unsigned)p.WIN) + 1u;
  const int grid = std::min(pl->num_sms, NT);
  const bool padw = pl->vf.pad_channel, elu = d.nl == IAF_NL_ELU;
  auto launch = [&](LyKernel lk, const IafLyParams& q, size_t smem) {
    const char* pe = getenv("IAF_PDL");
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(LY_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = (pe && pe[0] == '0') ? 0 : 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, lk, q) == cudaSuccess;
  };
  if (pl->fused) {
    IafLyParams q;
    memset(&q, 0, sizeof(q));
    q.t = p;
    for (int j = 0; j < 2; ++j) {
      IafTcStage& S_ = q.t.st[j];
      S_.whi = pl->whi[j]; S_.wlo = pl->wlo[j]; S_.bias = pl->bias[j]; S_.padw = pl->padw[j]; S_.wsinv = pl->wsinv[j];
      S_.hid_out = j == 0 ? a->hid_out[0] : nullptr;
      S_.cin = pl->cin[j]; S_.N = pl->N[j]; S_.K = pl->K[j];
    }
    q.t.n_stages = 2;
    q.t.sm_part = pl->fz_sm_part;
    q.in_mode = 0; q.first = 1; q.is_heads = 0;
    q.NB = LY_MAX_NB;
    q.sm_a = pl->fz_sm_a; q.sm_h = pl->fz_sm_h; q.sm_bias = pl->fz_sm_bias[0]; q.sm_bias1 = pl->fz_sm_bias[1];
    q.sm_part = pl->fz_sm_part; q.sm_acc = pl->fz_sm_acc; q.sm_b = pl->fz_sm_b[0]; q.sm_b1 = pl->fz_sm_b[1];
    q.b_chunk_bytes = LY_KC * 2 * pl->N[0] * 16; q.n_bchunks = (pl->K[0] / 16) / LY_KC;
    q.b_chunk_bytes1 = LY_KC * 2 * pl->N[1] * 16; q.n_bchunks1 = (pl->K[1] / 16) / LY_KC;
    q.stage_bytes = 2 * q.b_chunk_bytes;
    q.TS = TS; q.TO = TS;
    q.tl_enable = 1;
    if (!launch(fz_kernel_for(padw, a->mode, elu), q, pl->fz_smem)) return IAF_ERR_CUDA;
    if (n_launches) *n_launches = 1;
    return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
  }
  for (int j = 0; j < pl->n_stages; ++j) {
    IafLyParams q;
    memset(&q, 0, sizeof(q));
    q.t = p;
    q.TS = TC_TILE; q.TO = TC_TILE;
    IafTcStage& S_ = q.t.st[0];
    S_.whi = pl->whi[j]; S_.wlo = pl->wlo[j]; S_.bias = pl->bias[j];
    S_.padw = pl->padw[j]; S_.wsinv = pl->wsinv[j];
    S_.hid_out = (j < IAF_MAX_HIDDEN && j + 1 < pl->n_stages) ? a->hid_out[j] : nullptr;
    S_.cin = pl->cin[j]; S_.N = pl->N[j]; S_.K = pl->K[j];
    q.t.sm_part = pl->ly_sm_part[j];
    q.a_hi = j ? pl->img[(j - 1) & 1][0] : nullptr;
    q.a_lo = j ? pl->img[(j - 1) & 1][1] : nullptr;
    q.o_hi = pl->img[j & 1][0];
    q.o_lo = pl->img[j & 1][1];
    q.S_pad = pl->img_S_pad;
    q.in_mode = j ? 1 : 0;
    q.is_heads = j == pl->n_stages - 1;
    q.first = j == 0 && !q.is_heads;  // the first HIDDEN stage adds the context: never without one (ar.py:399-403)
    q.NB = pl->ly_NB[j];
    q.sm_a = pl->ly_sm_a[j]; q.sm_b = pl->ly_sm_b[j]; q.sm_bias = pl->ly_sm_bias[j]; q.sm_part = pl->ly_sm_part[j];
    q.sm_acc = pl->ly_sm_acc[j];
    q.b_chunk_bytes = LY_KC * 2 * pl->N[j] * 16;
    q.stage_bytes = pl->ly_stage[j];
    q.n_bchunks = (pl->K[j] / 16) / LY_KC;
    { const char* tls = getenv("IAF_TL_STAGE"); q.tl_enable = tls ? (atoi(tls) == j) : (j == pl->n_stages - 1); }
    if (!launch(ly_kernel_for(padw, a->mode, elu, pl->N[j]), q, pl->ly_smem[j])) return IAF_ERR_CUDA;
  }
  if (n_launches) *n_launches = pl->n_stages;
  return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
}

// ------------------------------------------------------------------------------------------
// Data gradient of the conv stack on the tensor cores (the "layers, top down" loop of iaf_bwd.cu).
//
// The transposed conv of layer j IS a hidden stage of iaf_ly_kernel: on the point-reflected stream (flip toggled) the
// taps of W^T are the same five slot shifts, so the gradient g (planes = the layer's packed output columns) goes in as an
// operand image, the transposed effective weights [5 * kin] x [cin] are the B operand, and the epilogue multiplies by
// nl'(h) (from the kept / recomputed activation h) and writes BOTH the fp32 gradient (weight-gradient kernel, context
// gradient) and the next operand image.  fp16 operand pairs need the gradient in fp16 range: each sample is scaled by a
// power of two chosen from its own max |g| at the heads (rows of the implicit GEMM are independent, so a per-sample
// scale is exact to undo and keeps the result independent of the rest of the batch).
// ------------------------------------------------------------------------------------------
struct IafDgPlan {
  iaf_desc_t d;
  int grad_flip;  // the gradient stream: the point reflection of the forward's (1 - IafVariantFlags::reflect)
  int n_stages;
  int kin[IAF_MAX_STAGES], nout[IAF_MAX_STAGES];  // dgrad of layer j: input planes (= packed columns of layer j), output channels (= cin of layer j)
  __nv_bfloat16* whi[IAF_MAX_STAGES];
  __nv_bfloat16* wlo[IAF_MAX_STAGES];
  float* zeros;  // bias table of the stages (the kernel adds it; the gradient has none): [5][maxn]
  int maxn;
  int sm_bias[IAF_MAX_STAGES], sm_part[IAF_MAX_STAGES], sm_acc[IAF_MAX_STAGES], sm_b[IAF_MAX_STAGES], stage[IAF_MAX_STAGES],
      NB[IAF_MAX_STAGES];
  size_t smem[IAF_MAX_STAGES];
  int MIR, WIN, MAXS, max_ch;
  __nv_bfloat16* img[2][2];  // ping-pong operand images [buffer][hi | lo]
  __nv_bfloat16* ximg[2];    // weight gradient: operand image of the current layer's input [hi | lo]
  int img_S_pad, scratch_B;
  float* wscale;             // [IAF_MAX_STAGES]: the power of two each stage's weight images carry
  float* amax;               // [B]
  float* bstep;              // [B][5][kin[last]]: per-sample bias / pad-channel sums of the fused step prologue
  int step_optin;            // the prologue kernel's dynamic shared memory limit has been raised
  int num_sms;
};

// Weight scale of a data-gradient stage: the power of two that brings the layer's largest effective weight into [32, 64)
// (dg_scale_from_amax).  The lo half of the fp16 split is subnormal below |w| ~ 2^-3 (absolute step 2^-24), so a
// small-gain layer (heads of gain 1e-3: |w| ~ 1e-4) would otherwise lose most of its 22 bits; the stage's epilogue
// divides it out again (exact).  One block: the weights of a stage are at most 5 x 256 x 256 floats.
__global__ void __launch_bounds__(1024) iaf_dg_wscale_kernel(const float4* __restrict__ w, int total4, float* wscale) {
  __shared__ float red[32];
  float m = 0.f;
  for (int i = threadIdx.x; i < total4; i += 1024) {
    const float4 v = __ldg(w + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = red[threadIdx.x];
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) *wscale = dg_scale_from_amax(m);
  }
}

__global__ void __launch_bounds__(256) iaf_dg_pack_kernel(const float* __restrict__ w, const float* __restrict__ wscale,
                                                          __nv_bfloat16* whi, __nv_bfloat16* wlo, int cin, int ncol) {
  // w: effective (masked, normalised) forward weights [tap][cin][ncol] fp32, times the stage's weight scale.  B operand of
  // the data gradient: K index [column / 16][tap][column % 16] (the layered kernel's K order), N index = ci; images
  // [K/8][N][8], fp16 hi / lo.
  const int total = IAF_NTAPS * cin * ncol;
  const float sw = __ldg(wscale);
  for (int i = blockIdx.x * 256 + threadIdx.x; i < total; i += gridDim.x * 256) {
    const int kc = i % ncol;
    const int ci = (i / ncol) % cin;
    const int t = i / (ncol * cin);
    const float vc = fminf(fmaxf(w[i] * sw, -65000.f), 65000.f);
    const __half hh = __float2half_rn(vc);
    const __half lh = __float2half_rn(vc - __half2float(hh));
    const int k = ((kc >> 4) * IAF_NTAPS + t) * 16 + (kc & 15);
    const size_t o = ((size_t)(k >> 3) * cin + ci) * 8 + (k & 7);
    whi[o] = __ushort_as_bfloat16(__half_as_ushort(hh));
    wlo[o] = __ushort_as_bfloat16(__half_as_ushort(lh));
  }
}

struct IafDgImageParams {
  const float* g;  // [B][planes][HW]
  float* amax;     // [B]
  __nv_bfloat16* o_hi;
  __nv_bfloat16* o_lo;
  int planes, H, W, Wp, SPS, HW, S_pad, flip;
  int S_end;       // slots [B * SPS, S_end) are zeroed by the extra block row (S_end = end of the zero tile past the last tile)
  int xmode, B;    // xmode 1: `g` is a layer INPUT for the weight gradient: scale c / s_n from the amax array (read only)
};
__global__ void __launch_bounds__(256) iaf_dg_image_kernel(const IafDgImageParams p) {
  // one block per sample: max |g| of the sample, then its slots of the operand image (pad slots as zeros)
  __shared__ float red[256];
  const int n = blockIdx.x, tid = threadIdx.x;
  if (n == p.B) {
    // one extra block row: zero the slots past the batch (up to the end of the zero tile).  The images outlive a call, a
    // smaller batch after a larger one must not leave the old samples' slots behind: the weight gradient sums over every
    // slot of every K tile
    const int nchunk_all = p.planes >> 3;
    const int c_lo = (int)((long long)nchunk_all * blockIdx.y / gridDim.y), c_hi = (int)((long long)nchunk_all * (blockIdx.y + 1) / gridDim.y);
    const int s0 = p.B * p.SPS, tail = p.S_end - s0;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    for (int i = tid; i < (c_hi - c_lo) * tail; i += 256) {
      const int c = c_lo + i / tail, r = i % tail;
      const size_t go = ((size_t)c * p.S_pad + s0 + r) * 8;
      *reinterpret_cast<uint4*>(p.o_hi + go) = zero;
      *reinterpret_cast<uint4*>(p.o_lo + go) = zero;
    }
    return;
  }
  const float* g = p.g + (size_t)n * p.planes * p.HW;
  float m = 0.f;
  if (p.xmode) {
    for (int i = tid; i < p.B; i += 256) m = fmaxf(m, p.amax[i]);  // the largest gradient of the batch
  } else {
    for (int i = tid; i < p.planes * p.HW; i += 256) m = fmaxf(m, fabsf(g[i]));
  }
  red[tid] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] = fmaxf(red[tid], red[tid + s]);
    __syncthreads();
  }
  m = red[0];
  if (tid == 0 && !p.xmode) p.amax[n] = m;
  // gradient image: s_n.  Input image of the weight gradient: c / s_n with c = the smallest scale of the batch (<= 1, a
  // power of two), so that every sample's X * G product carries the same factor c
  const float sc = p.xmode ? dg_scale_from_amax(m) / dg_scale_from_amax(p.amax[n]) : dg_scale_from_amax(m);
  const int nchunk_all = p.planes >> 3;
  // gridDim.y splits the chunk planes (input images of the weight gradient: up to 20 planes per sample)
  const int c_lo = (int)((long long)nchunk_all * blockIdx.y / gridDim.y), c_hi = (int)((long long)nchunk_all * (blockIdx.y + 1) / gridDim.y);
  const int nchunk = c_hi - c_lo;
  for (int i = tid; i < nchunk * p.SPS; i += 256) {
    const int c = c_lo + i / p.SPS, r = i % p.SPS;
    const int y = r / p.Wp, x = r - y * p.Wp;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (y < p.H && x < p.W) {
      const int pix = y * p.W + x;
      const int gp = p.flip ? p.HW - 1 - pix : pix;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = g[(size_t)(c * 8 + e) * p.HW + gp] * sc;
    }
    const size_t go = ((size_t)c * p.S_pad + (size_t)n * p.SPS + r) * 8;
    split_store8(v, reinterpret_cast<uint8_t*>(p.o_hi + go), reinterpret_cast<uint8_t*>(p.o_lo + go));
  }
}

void iaf_dg_plan_destroy(IafDgPlan* pl) {
  if (!pl) return;
  for (int j = 0; j < IAF_MAX_STAGES; ++j) {
    if (pl->whi[j]) cudaFree(pl->whi[j]);
    if (pl->wlo[j]) cudaFree(pl->wlo[j]);
  }
  if (pl->zeros) cudaFree(pl->zeros);
  if (pl->wscale) cudaFree(pl->wscale);
  if (pl->amax) cudaFree(pl->amax);
  if (pl->bstep) cudaFree(pl->bstep);
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b)
      if (pl->img[a][b]) cudaFree(pl->img[a][b]);
  for (int a = 0; a < 2; ++a)
    if (pl->ximg[a]) cudaFree(pl->ximg[a]);
  delete pl;
}

int iaf_dg_plan_create(IafDgPlan** out, const iaf_desc_t* d, const int* cin, const int* ncol, int n_stages) {
  *out = nullptr;
  const char* env = getenv("IAF_BWD_TC");
  if (env && env[0] == '0') return IAF_ERR_UNSUPPORTED;
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return IAF_ERR_CUDA;
  if (prop.major != 9) return IAF_ERR_UNSUPPORTED;  // wgmma: sm_90a
  const int Wp = d->W + 1;
  const int SPS = (d->H + 1) * Wp;
  const int MIR = tc_round_up(Wp + 1, 8);
  if (MIR > TC_TILE || n_stages > IAF_MAX_STAGES) return IAF_ERR_UNSUPPORTED;
  IafDgPlan* pl = new (std::nothrow) IafDgPlan();
  if (!pl) return IAF_ERR_BAD_ARG;
  memset(pl, 0, sizeof(*pl));
  pl->d = *d;
  pl->grad_flip = iaf_variant_flags(d->variant).reflect ? 0 : 1;
  pl->n_stages = n_stages;
  pl->MIR = MIR; pl->WIN = TC_TILE + MIR; pl->MAXS = (TC_TILE - 1) / SPS + 2;
  pl->num_sms = iaf_plan_num_sms(prop.multiProcessorCount);
  int maxn = 0;
  for (int j = 0; j < n_stages; ++j) {
    const int kin = ncol[j], N = cin[j];
    pl->kin[j] = kin; pl->nout[j] = N;
    pl->max_ch = std::max(pl->max_ch, std::max(kin, N));
    maxn = std::max(maxn, N);
    if (kin % 16 || N % 16 || kin > 256 || N > 32 * LY_MAX_NGW || N < 16) { iaf_dg_plan_destroy(pl); return IAF_ERR_UNSUPPORTED; }
    int off = 0;
    pl->sm_bias[j] = off; off += 5 * N * 4;
    off = tc_round_up(off, 16);
    pl->sm_part[j] = off; off += 2 * LY_PART_SETS * pl->MAXS * 4;
    off = tc_round_up(off, 16);
    pl->sm_acc[j] = off; off += TC_TILE * ly_acc_pitch(N) * 4;
    off = tc_round_up(off, 128);
    pl->sm_b[j] = off;
    const int slot = 2 * LY_KC * 2 * N * 16 + 4 * pl->WIN * 16;  // weight chunk hi+lo + A chunk pair hi+lo
    pl->stage[j] = slot;
    const int nb = (TC_SMEM_LIMIT - LY_B_SLACK - off) / slot;
    if (nb < 2) { iaf_dg_plan_destroy(pl); return IAF_ERR_UNSUPPORTED; }
    pl->NB[j] = std::min(nb, LY_MAX_NB);
    pl->smem[j] = (size_t)off + (size_t)pl->NB[j] * slot + LY_B_SLACK;
    const size_t wb = (size_t)IAF_NTAPS * kin * N * 2;
    if (cudaMalloc(&pl->whi[j], wb) != cudaSuccess || cudaMalloc(&pl->wlo[j], wb) != cudaSuccess) {
      iaf_dg_plan_destroy(pl);
      return IAF_ERR_CUDA;
    }
  }
  pl->maxn = maxn;
  // (zeros is filled on the first call's stream, by dg_ensure_scratch: the create has no stream to order it on)
  if (cudaMalloc(&pl->zeros, sizeof(float) * 5 * maxn) != cudaSuccess ||
      cudaMalloc(&pl->wscale, sizeof(float) * IAF_MAX_STAGES) != cudaSuccess) {
    iaf_dg_plan_destroy(pl);
    return IAF_ERR_CUDA;
  }
  cudaError_t oe = cudaSuccess;
  for (int j = 0; j < n_stages && oe == cudaSuccess; ++j)
    oe = iaf_smem_optin(ly_kernel_for(false, IAF_MODE_MULTICONV, d->nl == IAF_NL_ELU, pl->nout[j]));
  for (int k = 1; k <= WG_MAX_NP / 16 && oe == cudaSuccess; ++k)
    for (int w = 1; w <= 2 && oe == cudaSuccess; ++w) oe = iaf_smem_optin(wg_kernel_pick(k, w));
  if (oe != cudaSuccess) {
    iaf_dg_plan_destroy(pl);
    return IAF_ERR_CUDA;
  }
  if (Wp + 1 > WG_HALO) { iaf_dg_plan_destroy(pl); return IAF_ERR_UNSUPPORTED; }
  *out = pl;
  return IAF_OK;
}

// every zero-fill goes to the caller's stream, ahead of the kernels that read it
static int dg_ensure_scratch(IafDgPlan* pl, int B, cudaStream_t stream) {
  if (B <= pl->scratch_B) return IAF_OK;
  const int SPS = (pl->d.H + 1) * (pl->d.W + 1);
  if ((long long)B * SPS + TC_TILE >= (1LL << 31)) return IAF_ERR_UNSUPPORTED;
  const int NT = (B * SPS + TC_TILE - 1) / TC_TILE;
  pl->scratch_B = 0;  // a failure below must not leave the old size standing over freed buffers
  if (cudaMemsetAsync(pl->zeros, 0, sizeof(float) * 5 * pl->maxn, stream) != cudaSuccess) return IAF_ERR_CUDA;
  pl->img_S_pad = (NT + 1) * TC_TILE;  // one zero tile past the end: windows of the last tile read into it
  const size_t bytes = (size_t)(pl->max_ch / 8) * pl->img_S_pad * 16;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      if (pl->img[a][b]) cudaFree(pl->img[a][b]);
      pl->img[a][b] = nullptr;
      if (cudaMalloc(&pl->img[a][b], bytes) != cudaSuccess) return IAF_ERR_CUDA;
      if (cudaMemsetAsync(pl->img[a][b], 0, bytes, stream) != cudaSuccess) return IAF_ERR_CUDA;
    }
  for (int a = 0; a < 2; ++a) {
    if (pl->ximg[a]) cudaFree(pl->ximg[a]);
    pl->ximg[a] = nullptr;
    if (cudaMalloc(&pl->ximg[a], bytes) != cudaSuccess) return IAF_ERR_CUDA;
    if (cudaMemsetAsync(pl->ximg[a], 0, bytes, stream) != cudaSuccess) return IAF_ERR_CUDA;
  }
  if (pl->amax) cudaFree(pl->amax);
  if (pl->bstep) cudaFree(pl->bstep);
  pl->amax = pl->bstep = nullptr;
  if (cudaMalloc(&pl->amax, sizeof(float) * (size_t)B) != cudaSuccess) return IAF_ERR_CUDA;
  if (cudaMalloc(&pl->bstep, sizeof(float) * (size_t)B * 5 * pl->kin[pl->n_stages - 1]) != cudaSuccess) return IAF_ERR_CUDA;
  pl->scratch_B = B;
  return IAF_OK;
}

// gradient at the heads (fp32 [B][kin[last]][HW]) -> per-sample scale + operand image 0
int iaf_dg_begin(IafDgPlan* pl, const float* g_heads, int B, cudaStream_t stream) {
  const iaf_desc_t& d = pl->d;
  int st = dg_ensure_scratch(pl, B, stream);
  if (st != IAF_OK) return st;
  IafDgImageParams q;
  memset(&q, 0, sizeof(q));
  q.g = g_heads; q.amax = pl->amax; q.o_hi = pl->img[0][0]; q.o_lo = pl->img[0][1];
  q.planes = pl->kin[pl->n_stages - 1]; q.H = d.H; q.W = d.W; q.Wp = d.W + 1; q.SPS = (d.H + 1) * (d.W + 1);
  q.HW = d.H * d.W; q.S_pad = pl->img_S_pad;
  q.flip = pl->grad_flip;  // the data gradient runs on the point-reflected stream of the forward
  q.xmode = 0; q.B = B;
  // gridDim.y splits the image planes; every y-block recomputes the sample's max (L2 hits) and writes the same value
  q.S_end = ((B * q.SPS + TC_TILE - 1) / TC_TILE + 1) * TC_TILE;
  iaf_dg_image_kernel<<<dim3(B + 1, std::max(1, q.planes / 16)), 256, 0, stream>>>(q);
  return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
}

// data gradient of layer j: image `in_buf` (kin[j] planes) -> fp32 `out` [B][nout[j]][HW] (x nl'(hprev) when hprev is
// given; accumulated into `out` when it is not: the stack input) and, when `write_image`, the next operand image
int iaf_dg_stage(IafDgPlan* pl, int j, const float* w_packed, int in_buf, const float* hprev, float* out, int write_image,
                 int B, cudaStream_t stream) {
  const iaf_desc_t& d = pl->d;
  const int kin = pl->kin[j], N = pl->nout[j];
  {
    const int total = IAF_NTAPS * N * kin;
    iaf_dg_wscale_kernel<<<1, 1024, 0, stream>>>(reinterpret_cast<const float4*>(w_packed), total / 4, pl->wscale + j);
    iaf_dg_pack_kernel<<<std::min(592, (total + 255) / 256), 256, 0, stream>>>(w_packed, pl->wscale + j, pl->whi[j],
                                                                              pl->wlo[j], N, kin);
    if (cudaGetLastError() != cudaSuccess) return IAF_ERR_CUDA;
  }
  const int SPS = (d.H + 1) * (d.W + 1);
  const int S = B * SPS;
  const int NT = (S + TC_TILE - 1) / TC_TILE;
  IafLyParams q;
  memset(&q, 0, sizeof(q));
  IafTcParams& p = q.t;
  p.ctx = hprev;
  p.n_stages = 1;
  IafTcStage& S_ = p.st[0];
  S_.whi = pl->whi[j]; S_.wlo = pl->wlo[j]; S_.bias = pl->zeros; S_.padw = nullptr;
  S_.hid_out = out;
  S_.cin = kin; S_.N = N; S_.K = IAF_NTAPS * kin;
  p.B = B; p.C = d.n_z; p.H = d.H; p.W = d.W; p.Wp = d.W + 1; p.SPS = SPS; p.HW = d.H * d.W;
  p.S = S; p.NT = NT;
  p.MIR = pl->MIR; p.WIN = pl->WIN; p.MAXS = pl->MAXS; p.sm_part = pl->sm_part[j];
  p.flip = pl->grad_flip;
  p.nl = d.nl; p.scale = 0.1f;
  p.mg_sps = (unsigned)((1ULL << 32) / (unsigned)SPS) + 1u;
  p.mg_wp = (unsigned)((1ULL << 32) / (unsigned)p.Wp) + 1u;
  p.mg_win = (unsigned)((1ULL << 32) / (unsigned)p.WIN) + 1u;
  q.a_hi = pl->img[in_buf][0]; q.a_lo = pl->img[in_buf][1];
  q.o_hi = write_image ? pl->img[in_buf ^ 1][0] : nullptr;
  q.o_lo = write_image ? pl->img[in_buf ^ 1][1] : nullptr;
  q.S_pad = pl->img_S_pad;
  q.in_mode = 1;
  q.is_heads = 0;
  q.first = hprev ? 1 : 0;
  q.NB = pl->NB[j];
  q.sm_a = 0; q.sm_b = pl->sm_b[j]; q.sm_bias = pl->sm_bias[j]; q.sm_part = pl->sm_part[j]; q.sm_acc = pl->sm_acc[j];
  q.b_chunk_bytes = LY_KC * 2 * N * 16;
  q.stage_bytes = pl->stage[j];
  q.n_bchunks = kin / 16;
  q.bwd = hprev ? 1 : 2;
  q.amax = pl->amax;
  q.wscale = pl->wscale + j;
  q.TS = TC_TILE; q.TO = TC_TILE;
  LyKernel lk = ly_kernel_for(false, IAF_MODE_MULTICONV, d.nl == IAF_NL_ELU, N);
  const int grid = std::min(pl->num_sms, NT);
  lk<<<grid, LY_THREADS, pl->smem[j], stream>>>(q);
  return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
}

// weight gradient of layer j: X = the layer's input (fp32 [B][nout[j]][HW]), G = operand image `g_buf` (kin[j] planes,
// the input of data-gradient stage j).  Partials go to part[group][...] (stride part_stride floats); *ng_used groups.
int iaf_wg_run(IafDgPlan* pl, int j, const float* x, int g_buf, float* part, int part_stride, int ng_max, int B,
               cudaStream_t stream, int* ng_used) {
  const iaf_desc_t& d = pl->d;
  const int cin = pl->nout[j], ncol = pl->kin[j];
  const int SPS = (d.H + 1) * (d.W + 1);
  {
    IafDgImageParams q;
    memset(&q, 0, sizeof(q));
    q.g = x; q.amax = pl->amax; q.o_hi = pl->ximg[0]; q.o_lo = pl->ximg[1];
    q.planes = cin; q.H = d.H; q.W = d.W; q.Wp = d.W + 1; q.SPS = SPS; q.HW = d.H * d.W; q.S_pad = pl->img_S_pad;
    q.flip = pl->grad_flip;
    q.xmode = 1; q.B = B;
    q.S_end = ((B * SPS + TC_TILE - 1) / TC_TILE + 1) * TC_TILE;
    iaf_dg_image_kernel<<<dim3(B + 1, std::max(1, cin / 32)), 256, 0, stream>>>(q);
    if (cudaGetLastError() != cudaSuccess) return IAF_ERR_CUDA;
  }
  IafWgTcParams q;
  memset(&q, 0, sizeof(q));
  q.x_hi = pl->ximg[0]; q.x_lo = pl->ximg[1];
  q.g_hi = pl->img[g_buf][0]; q.g_lo = pl->img[g_buf][1];
  q.part = part; q.amax = pl->amax;
  q.B = B; q.cin = cin; q.ncol = ncol; q.S_pad = pl->img_S_pad; q.Wp = d.W + 1;
  int Np = 16;
  for (int c = 16; c <= WG_MAX_NP; c += 16)
    if (ncol % c == 0) Np = c;
  q.Np = Np; q.n_np = ncol / Np; q.n_mb = (cin + 127) / 128;
  const int NT = (B * SPS + TC_TILE - 1) / TC_TILE;
  q.NTK = NT * (TC_TILE / WG_KT);
  const int ntiles = q.n_mb * q.n_np;
  q.NG = std::max(1, std::min(std::min(ng_max, q.NTK), pl->num_sms / ntiles));
  q.part_stride = part_stride;
  q.xplanes = std::min(16, cin / 8); q.gplanes = Np / 8;
  q.xa_bytes = 2 * q.xplanes * WG_KT * 16;
  q.stage_bytes = q.xa_bytes + 2 * q.gplanes * (WG_KT + WG_HALO) * 16;
  const int slack = 16 * WG_KT * 16 + 1024;  // the M = 128 descriptor walks 16 planes whatever the layer has: stay inside the allocation
  q.n_stages = std::min(WG_MAX_STAGES, (TC_SMEM_LIMIT - slack) / q.stage_bytes);
  if (q.n_stages < 2) return IAF_ERR_UNSUPPORTED;
  const size_t smem = (size_t)q.n_stages * q.stage_bytes + slack;
  const int nwg = cin > 64 ? 2 : 1;
  wg_kernel_pick(q.Np / 16, nwg)<<<ntiles * q.NG, WG_THREADS(nwg), smem, stream>>>(q);
  if (ng_used) *ng_used = q.NG;
  return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
}

struct IafDgStepParams {
  const float* z_out; const float* logsd; const float* g_zout; const float* g_logsd; const float* g_logdet;
  float* g_z; float* hb; float* bstep; float* amax;
  __nv_bfloat16* o_hi; __nv_bfloat16* o_lo;
  int B, C, cp, head_pad, H, W, Wp, SPS, HW, S_pad, S_end, fwd_flip, img_flip;
  float scale;
  const float* g_logps; const float* g_logp_bc; const float* g_logp;  // LOGP: the MADE prior density's upstream, nullable
};

// ------------------------------------------------------------------------------------------
// Fused prologue of the tensor-core backward of the STEP entry with kept activations: what iaf_bwd_affine_kernel,
// iaf_dg_image_kernel and the heads' iaf_bwd_bias_kernel do in three passes over [B][2 n_z][HW], in one: a block per sample
// forms g_m, g_s (models.py:282-285 differentiated) in shared memory, writes the direct term of g_z, the sample's max and
// scale, its bias / pad-channel column sums, and the scaled operand image of the heads' gradient.
// LOGP: the MADE prior's density (logps = -0.5 log 2pi - arw_logsd - 0.5 z'^2) with the upstream
// G = g_logps + g_logp_bc[b,c] + g_logp[b] in place of the step's: g_z' = -z' G, g_arw_logsd = -G.
// ------------------------------------------------------------------------------------------
template <bool LOGP>
__global__ void __launch_bounds__(256) iaf_dg_step_kernel(const __grid_constant__ IafDgStepParams p) {
  extern __shared__ float sg[];  // [cp][HW]
  __shared__ float red[256];
  const int n = blockIdx.x, tid = threadIdx.x, HW = p.HW;
  if (n == p.B) {  // zero the image slots past the batch (see iaf_dg_image_kernel)
    const int nchunk = p.cp >> 3;
    const int s0 = p.B * p.SPS, tail = p.S_end - s0;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    for (int i = tid; i < nchunk * tail; i += 256) {
      const size_t go = ((size_t)(i / tail) * p.S_pad + s0 + i % tail) * 8;
      *reinterpret_cast<uint4*>(p.o_hi + go) = zero;
      *reinterpret_cast<uint4*>(p.o_lo + go) = zero;
    }
    return;
  }
  for (int i = tid; i < p.cp * HW; i += 256) sg[i] = 0.f;
  __syncthreads();
  float m = 0.f;
  const float gld = p.g_logdet ? __ldg(p.g_logdet + n) : 0.f;
  for (int i = tid; i < p.C * HW; i += 256) {
    const int c = i / HW, gp = i - c * HW;
    const int mcol = (c >> 2) * 8 + (c & 3), scol = mcol + 4;
    const size_t e = ((size_t)n * p.C + c) * HW + gp;
    float gzo, gs, ex, zn;
    if (LOGP) {
      ex = expf(-__ldg(p.logsd + e));
      zn = __ldg(p.z_out + e);
      float G = 0.f;
      if (p.g_logps) G += __ldg(p.g_logps + e);
      if (p.g_logp_bc) G += __ldg(p.g_logp_bc + (size_t)n * p.C + c);
      if (p.g_logp) G += __ldg(p.g_logp + n);
      gzo = -zn * G;
      gs = -p.scale * zn * gzo - p.scale * G;
    } else {
      ex = expf(-__ldg(p.logsd + e)); zn = __ldg(p.z_out + e); gzo = __ldg(p.g_zout + e);
      gs = -p.scale * zn * gzo;
      if (p.g_logsd) gs += p.scale * __ldg(p.g_logsd + e);
      gs -= p.scale * gld;
    }
    const float gm = -p.scale * ex * gzo;
    sg[mcol * HW + gp] = gm;
    sg[scol * HW + gp] = gs;
    p.g_z[e] = ex * gzo;
    if (p.hb) {
      p.hb[((size_t)n * p.cp + mcol) * HW + gp] = gm;
      p.hb[((size_t)n * p.cp + scol) * HW + gp] = gs;
    }
    m = fmaxf(m, fmaxf(fabsf(gm), fabsf(gs)));
  }
  red[tid] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] = fmaxf(red[tid], red[tid + s]);
    __syncthreads();
  }
  m = red[0];
  if (tid == 0) p.amax[n] = m;
  const float sc = dg_scale_from_amax(m);
  // column sums of this sample (fixed order: lane-strided, xor-shuffle tree); warp w owns columns w, w + 8, ...
  {
    const int warp = tid >> 5, lane = tid & 31;
    for (int col = warp; col < p.cp; col += 8) {
      float s5[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
      for (int gp = lane; gp < HW; gp += 32) {
        const float v = sg[col * HW + gp];
        const int pix = p.fwd_flip ? HW - 1 - gp : gp;  // logical position of this memory pixel
        const int y = pix / p.W, x = pix - y * p.W;
        const bool byH = (y == p.H - 1), bx0 = (x == 0), bxW = (x == p.W - 1);
        s5[0] += v;
        s5[1] += bxW ? v : 0.f;
        s5[2] += (byH || bx0) ? v : 0.f;
        s5[3] += byH ? v : 0.f;
        s5[4] += (byH || bxW) ? v : 0.f;
      }
#pragma unroll
      for (int t = 0; t < 5; ++t) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s5[t] += __shfl_xor_sync(0xffffffffu, s5[t], o);
        if (lane == 0) p.bstep[((size_t)n * 5 + t) * p.cp + col] = s5[t];
      }
    }
  }
  // operand image of the sample (point-reflected stream of the forward), pad slots as zeros
  const int nchunk = p.cp >> 3;
  for (int i = tid; i < nchunk * p.SPS; i += 256) {
    const int c = i / p.SPS, r = i - c * p.SPS;
    const int y = r / p.Wp, x = r - y * p.Wp;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (y < p.H && x < p.W) {
      const int pix = y * p.W + x;
      const int gp = p.img_flip ? HW - 1 - pix : pix;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = sg[(c * 8 + e) * HW + gp] * sc;
    }
    const size_t go = ((size_t)c * p.S_pad + (size_t)n * p.SPS + r) * 8;
    split_store8(v, reinterpret_cast<uint8_t*>(p.o_hi + go), reinterpret_cast<uint8_t*>(p.o_lo + go));
  }
}

bool iaf_dg_step_supported(const IafDgPlan* pl) {
  const char* e = getenv("IAF_BWD_FUSED_PROLOGUE");
  if (e && e[0] == '0') return false;
  return (size_t)pl->kin[pl->n_stages - 1] * pl->d.H * pl->d.W * 4 <= 160 * 1024;
}

// STEP entry with kept activations: g_z (direct term), per-sample scale, bias sums (-> *bias_partials, [B][5][cp]) and the
// operand image 0 of the heads' gradient in one launch.  hb (fp32 heads gradient) is optional.
static int dg_begin_step(IafDgPlan* pl, IafDgStepParams& q, bool logp, float* g_z, float* hb, int head_pad, int B,
                         cudaStream_t stream, const float** bias_partials) {
  const iaf_desc_t& d = pl->d;
  int st = dg_ensure_scratch(pl, B, stream);
  if (st != IAF_OK) return st;
  if (!pl->step_optin) {
    if (iaf_smem_optin(iaf_dg_step_kernel<false>) != cudaSuccess) return IAF_ERR_CUDA;
    if (iaf_smem_optin(iaf_dg_step_kernel<true>) != cudaSuccess) return IAF_ERR_CUDA;
    pl->step_optin = 1;
  }
  q.g_z = g_z; q.hb = hb; q.bstep = pl->bstep; q.amax = pl->amax;
  q.o_hi = pl->img[0][0]; q.o_lo = pl->img[0][1];
  q.B = B; q.C = d.n_z; q.cp = pl->kin[pl->n_stages - 1]; q.head_pad = head_pad;
  q.H = d.H; q.W = d.W; q.Wp = d.W + 1; q.SPS = (d.H + 1) * (d.W + 1); q.HW = d.H * d.W;
  q.S_pad = pl->img_S_pad;
  q.S_end = ((B * q.SPS + TC_TILE - 1) / TC_TILE + 1) * TC_TILE;
  q.img_flip = pl->grad_flip;
  q.fwd_flip = q.img_flip ? 0 : 1;
  q.scale = 0.1f;
  if (logp) iaf_dg_step_kernel<true><<<B + 1, 256, (size_t)q.cp * q.HW * 4, stream>>>(q);
  else iaf_dg_step_kernel<false><<<B + 1, 256, (size_t)q.cp * q.HW * 4, stream>>>(q);
  if (bias_partials) *bias_partials = pl->bstep;
  return cudaGetLastError() == cudaSuccess ? IAF_OK : IAF_ERR_CUDA;
}

int iaf_dg_begin_step(IafDgPlan* pl, const float* z_out, const float* logsd, const float* g_zout, const float* g_logsd,
                      const float* g_logdet, float* g_z, float* hb, int head_pad, int B, cudaStream_t stream,
                      const float** bias_partials) {
  IafDgStepParams q;
  memset(&q, 0, sizeof(q));
  q.z_out = z_out; q.logsd = logsd; q.g_zout = g_zout; q.g_logsd = g_logsd; q.g_logdet = g_logdet;
  return dg_begin_step(pl, q, false, g_z, hb, head_pad, B, stream, bias_partials);
}

int iaf_dg_begin_step_logp(IafDgPlan* pl, const float* z_out, const float* logsd, const float* g_logps,
                           const float* g_logp_bc, const float* g_logp, float* g_z, float* hb, int head_pad, int B,
                           cudaStream_t stream, const float** bias_partials) {
  IafDgStepParams q;
  memset(&q, 0, sizeof(q));
  q.z_out = z_out; q.logsd = logsd; q.g_logps = g_logps; q.g_logp_bc = g_logp_bc; q.g_logp = g_logp;
  return dg_begin_step(pl, q, true, g_z, hb, head_pad, B, stream, bias_partials);
}
