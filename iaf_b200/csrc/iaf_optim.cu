// The reference's Adamax update and weight average (include/iaf_b200.h, iaf_adamax_step), and its Eve update
// (iaf_eve_step), each over a whole parameter set in one launch.
//
// The tensor table travels by value in the kernel's parameter space (__grid_constant__: read in place from the constant
// bank, never copied to local memory), so a step needs no device allocation and no host->device copy and can be
// captured into a CUDA graph.  Each entry owns ceil(numel / IAF_OPT_TILE) consecutive CTAs; block0[i] is entry i's
// first, and a CTA finds its entry by binary search.  A tile is loaded as float4 when every one of its streams is
// 16-byte aligned (the tile starts are multiples of 4 elements, so a tensor's base pointers decide), element by element
// otherwise: a view at an odd storage offset takes the scalar loop.
//
// Per element the arithmetic is the fixed sequence of correctly rounded fp32 operations include/iaf_b200.h lists, spelled
// with the _rn intrinsics so that nvcc cannot contract a multiply and an add into an FMA.
#include "iaf_common.h"

#ifdef IAF_EMU
// host emulation: plain fp32 operations (x86-64 g++ without -mfma does not contract them)
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
#endif

#define IAF_OPT_THREADS 256
#define IAF_OPT_TILE (IAF_OPT_THREADS * 16)  // elements per CTA: four float4 per thread

struct IafAdamaxParams {
  iaf_adamax_tensor_t t[IAF_ADAMAX_MAX_TENSORS];
  int block0[IAF_ADAMAX_MAX_TENSORS];
  float* mom1;
  float* mom_max;
  float* avg;
  int n;
  float grad_scale;
  // TF:     c0 = lr, c1 = b1, c2 = 1 - b1 (fp32), c3 = b2, c4 = 1e-8, c5 = 1 - avg_decay
  // Theano: c0 = -lr, c1 = 1 - b1, c2 = b1, c3 = 1 - b2, c4 = 1e-8, c5 = 1 - avg_decay, c6 = avg_decay
  float c[7];
};
// the parameter space of a launch is 32764 bytes (CUDA 12.1+, Volta and newer)
static_assert(sizeof(IafAdamaxParams) <= 32764, "the tensor table must fit in one launch's parameter space");

// One element.  HAS_G false: TF's skipped tensor (only the average moves) or Theano's zero gradient.
template <int RULE, bool HAS_G>
__device__ __forceinline__ void adamax_elem(const IafAdamaxParams& p, float& w, float g, float& m1, float& mx,
                                            float& a) {
  const float* c = p.c;
  if (RULE == IAF_ADAMAX_TF) {
    a = __fsub_rn(a, __fmul_rn(__fsub_rn(a, w), c[5]));  // avg -= (avg - p) (1 - decay), p before the update
    if (!HAS_G) return;
    g = __fmul_rn(g, p.grad_scale);
    m1 = __fadd_rn(__fmul_rn(c[1], m1), __fmul_rn(c[2], g));   // v = b1 v + (1 - b1) g
    mx = fmaxf(__fadd_rn(__fmul_rn(c[3], mx), c[4]), fabsf(g));  // m = max(b2 m + eps, |g|)
    w = __fsub_rn(w, __fmul_rn(c[0], __fdiv_rn(m1, mx)));     // p -= lr (v / m)
  } else {
    g = HAS_G ? __fmul_rn(g, p.grad_scale) : 0.f;
    a = __fadd_rn(__fmul_rn(c[5], w), __fmul_rn(c[6], a));     // avg = b2 p + (1 - b2) avg, p before the update
    m1 = __fadd_rn(__fmul_rn(c[1], m1), __fmul_rn(c[2], g));   // mom1 = (1 - b1) mom1 + b1 g
    mx = fmaxf(__fmul_rn(c[3], mx), __fadd_rn(fabsf(g), c[4]));  // max = max((1 - b2) max, |g| + 1e-8)
    w = __fadd_rn(w, __fdiv_rn(__fmul_rn(c[0], m1), mx));     // p = p + (alpha mom1) / max, alpha = -lr
  }
}

// TF's skipped tensor touches only p (read) and avg
template <int RULE, bool HAS_G>
__device__ __forceinline__ void adamax_tile(const IafAdamaxParams& p, float* w, const float* g, float* m1, float* mx,
                                            float* a, int len) {
  const bool avg_only = RULE == IAF_ADAMAX_TF && !HAS_G;
  const uintptr_t bits = (uintptr_t)w | (uintptr_t)g | (uintptr_t)m1 | (uintptr_t)mx | (uintptr_t)a;
  int done = 0;
  if ((bits & 15) == 0) {
    const int nv = len >> 2;
    for (int i = threadIdx.x; i < nv; i += IAF_OPT_THREADS) {
      float4 W = reinterpret_cast<const float4*>(w)[i];
      float4 A = reinterpret_cast<const float4*>(a)[i];
      float4 G = make_float4(0.f, 0.f, 0.f, 0.f), M = G, X = G;
      if (HAS_G) G = reinterpret_cast<const float4*>(g)[i];
      if (!avg_only) {
        M = reinterpret_cast<const float4*>(m1)[i];
        X = reinterpret_cast<const float4*>(mx)[i];
      }
      adamax_elem<RULE, HAS_G>(p, W.x, G.x, M.x, X.x, A.x);
      adamax_elem<RULE, HAS_G>(p, W.y, G.y, M.y, X.y, A.y);
      adamax_elem<RULE, HAS_G>(p, W.z, G.z, M.z, X.z, A.z);
      adamax_elem<RULE, HAS_G>(p, W.w, G.w, M.w, X.w, A.w);
      reinterpret_cast<float4*>(a)[i] = A;
      if (!avg_only) {
        reinterpret_cast<float4*>(w)[i] = W;
        reinterpret_cast<float4*>(m1)[i] = M;
        reinterpret_cast<float4*>(mx)[i] = X;
      }
    }
    done = nv << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += IAF_OPT_THREADS) {
    float W = w[i], A = a[i], G = HAS_G ? g[i] : 0.f, M = avg_only ? 0.f : m1[i], X = avg_only ? 0.f : mx[i];
    adamax_elem<RULE, HAS_G>(p, W, G, M, X, A);
    a[i] = A;
    if (!avg_only) {
      w[i] = W;
      m1[i] = M;
      mx[i] = X;
    }
  }
}

// The table entry CTA b works on: the last one whose first CTA is <= b.
__device__ __forceinline__ int iaf_opt_entry(const int* block0, int n, int b) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (block0[mid] <= b) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <int RULE>
__global__ void __launch_bounds__(IAF_OPT_THREADS) iaf_adamax_kernel(const __grid_constant__ IafAdamaxParams p) {
  const int b = blockIdx.x;
  const int lo = iaf_opt_entry(p.block0, p.n, b);
  const iaf_adamax_tensor_t& T = p.t[lo];
  const int64_t start = (int64_t)(b - p.block0[lo]) * IAF_OPT_TILE;
  const int64_t rem = T.numel - start;
  const int len = rem < IAF_OPT_TILE ? (int)rem : IAF_OPT_TILE;
  const int64_t s = T.offset + start;
  if (T.grad)
    adamax_tile<RULE, true>(p, T.param + start, T.grad + start, p.mom1 + s, p.mom_max + s, p.avg + s, len);
  else
    adamax_tile<RULE, false>(p, T.param + start, nullptr, p.mom1 + s, p.mom_max + s, p.avg + s, len);
}

// The table in chunks of IAF_ADAMAX_MAX_TENSORS entries (fewer where the grid's x extent runs out), one launch(blocks)
// each with p.t / p.block0 / p.n filled in.  *launches counts the launches made.
template <class P, class Launch>
static int iaf_opt_launch_chunks(P& p, const iaf_adamax_tensor_t* tensors_host, int n_tensors, uint64_t* launches,
                                 const char* what, Launch launch) {
  for (int i0 = 0; i0 < n_tensors;) {
    int n = 0, blocks = 0;
    for (; i0 + n < n_tensors && n < IAF_ADAMAX_MAX_TENSORS; ++n) {
      const int64_t nb = (tensors_host[i0 + n].numel + IAF_OPT_TILE - 1) / IAF_OPT_TILE;
      if (nb > 0x7fffffff - (int64_t)blocks) break;  // the grid's x extent; the next launch takes the rest
      p.t[n] = tensors_host[i0 + n];
      p.block0[n] = blocks;
      blocks += (int)nb;
    }
    p.n = n;
    launch(blocks);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return iaf_record_cuda_error(e, what);
    ++*launches;
    i0 += n;
  }
  return IAF_OK;
}

// The launcher behind iaf_adamax_step (iaf_capi.cu validates the arguments first): the constants as the rule rounds
// them, then the table in chunks, one launch each.
static int iaf_adamax_launch(int rule, const iaf_adamax_tensor_t* tensors_host, int n_tensors, float* mom1,
                             float* mom_max, float* avg, double lr, double beta1, double beta2, double avg_decay,
                             float grad_scale, void* stream, uint64_t* launches) {
  IafAdamaxParams p;
  p.mom1 = mom1;
  p.mom_max = mom_max;
  p.avg = avg;
  p.grad_scale = grad_scale;
  for (float& v : p.c) v = 0.f;
  if (rule == IAF_ADAMAX_TF) {  // adamax.py:41-47: constants cast to fp32, 1. - beta1_t computed in fp32
    const float b1 = (float)beta1;
    p.c[0] = (float)lr;
    p.c[1] = b1;
    p.c[2] = 1.f - b1;
    p.c[3] = (float)beta2;
    p.c[4] = 1e-8f;
    p.c[5] = (float)(1.0 - avg_decay);  // assign_moving_average: convert_to_tensor(1.0 - decay)
  } else {  // optim.py:116-122: python float constants, cast to floatX
    p.c[0] = (float)(-lr);
    p.c[1] = (float)(1.0 - beta1);
    p.c[2] = (float)beta1;
    p.c[3] = (float)(1.0 - beta2);
    p.c[4] = 1e-8f;
    p.c[5] = (float)(1.0 - avg_decay);
    p.c[6] = (float)avg_decay;
  }

  cudaStream_t st = (cudaStream_t)stream;
  return iaf_opt_launch_chunks(p, tensors_host, n_tensors, launches, "iaf_adamax_kernel", [&](int blocks) {
    if (rule == IAF_ADAMAX_TF)
      IAF_LAUNCH(iaf_adamax_kernel<IAF_ADAMAX_TF>, blocks, IAF_OPT_THREADS, 0, st, p);
    else
      IAF_LAUNCH(iaf_adamax_kernel<IAF_ADAMAX_THEANO>, blocks, IAF_OPT_THREADS, 0, st, p);
  });
}

// ---------------------------------------------------------------------------------------------------------------------
// Eve (include/iaf_b200.h, iaf_eve_step): the same table, tiling and entry search as the Adamax kernel, with a parameter
// struct of its own.  The previous delta is not read: the new one does not depend on it, and the lookahead it enters is
// the one this kernel wrote last step.  So an element reads w, g, mom1, max and avg and writes all but g plus w'.
struct IafEveParams {
  iaf_adamax_tensor_t t[IAF_ADAMAX_MAX_TENSORS];
  int block0[IAF_ADAMAX_MAX_TENSORS];
  float* mom1;
  float* mom_max;
  float* delta;
  float* avg;
  float* lookahead;
  int n;
  float grad_scale;
  // c0 = alpha = -lr, c1 = 1 - b1, c2 = b1, c3 = 1 - b2, c4 = 1e-8, c5 = b3, c6 = 1 - b3, c7 = (1 - b1) / b1
  float c[8];
};
static_assert(sizeof(IafEveParams) <= 32764, "the tensor table must fit in one launch's parameter space");

// One element; g is 0 for a NULL gradient.  d receives the new delta, la the next step's lookahead.
__device__ __forceinline__ void eve_elem(const IafEveParams& p, float& w, float g, float& m1, float& mx, float& d,
                                         float& a, float& la) {
  const float* c = p.c;
  g = __fmul_rn(g, p.grad_scale);
  a = __fadd_rn(__fmul_rn(c[5], w), __fmul_rn(c[6], a));     // avg = b3 w + (1 - b3) avg, w before the update
  m1 = __fadd_rn(__fmul_rn(c[1], m1), __fmul_rn(c[2], g));   // mom1 = (1 - b1) mom1 + b1 g
  mx = fmaxf(__fmul_rn(c[3], mx), __fadd_rn(fabsf(g), c[4]));  // max = max((1 - b2) max, |g| + 1e-8)
  d = __fdiv_rn(__fmul_rn(c[0], m1), mx);                    // delta = (alpha mom1) / max
  w = __fadd_rn(w, d);                                       // w = w + delta
  la = __fadd_rn(w, __fmul_rn(c[7], d));                     // w' = w + (1 - b1) / b1 delta, for the next step
}

template <bool HAS_G>
__device__ __forceinline__ void eve_tile(const IafEveParams& p, float* w, const float* g, float* m1, float* mx,
                                         float* d, float* a, float* la, int len) {
  const uintptr_t bits = (uintptr_t)w | (uintptr_t)g | (uintptr_t)m1 | (uintptr_t)mx | (uintptr_t)d | (uintptr_t)a |
                         (uintptr_t)la;
  int done = 0;
  if ((bits & 15) == 0) {
    const int nv = len >> 2;
    for (int i = threadIdx.x; i < nv; i += IAF_OPT_THREADS) {
      float4 W = reinterpret_cast<const float4*>(w)[i];
      float4 M = reinterpret_cast<const float4*>(m1)[i];
      float4 X = reinterpret_cast<const float4*>(mx)[i];
      float4 A = reinterpret_cast<const float4*>(a)[i];
      float4 G = make_float4(0.f, 0.f, 0.f, 0.f), D, L;
      if (HAS_G) G = reinterpret_cast<const float4*>(g)[i];
      eve_elem(p, W.x, G.x, M.x, X.x, D.x, A.x, L.x);
      eve_elem(p, W.y, G.y, M.y, X.y, D.y, A.y, L.y);
      eve_elem(p, W.z, G.z, M.z, X.z, D.z, A.z, L.z);
      eve_elem(p, W.w, G.w, M.w, X.w, D.w, A.w, L.w);
      reinterpret_cast<float4*>(w)[i] = W;
      reinterpret_cast<float4*>(m1)[i] = M;
      reinterpret_cast<float4*>(mx)[i] = X;
      reinterpret_cast<float4*>(d)[i] = D;
      reinterpret_cast<float4*>(a)[i] = A;
      reinterpret_cast<float4*>(la)[i] = L;
    }
    done = nv << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += IAF_OPT_THREADS) {
    float W = w[i], M = m1[i], X = mx[i], A = a[i], D, L;
    eve_elem(p, W, HAS_G ? g[i] : 0.f, M, X, D, A, L);
    w[i] = W;
    m1[i] = M;
    mx[i] = X;
    d[i] = D;
    a[i] = A;
    la[i] = L;
  }
}

__global__ void __launch_bounds__(IAF_OPT_THREADS) iaf_eve_kernel(const __grid_constant__ IafEveParams p) {
  const int b = blockIdx.x;
  const int lo = iaf_opt_entry(p.block0, p.n, b);
  const iaf_adamax_tensor_t& T = p.t[lo];
  const int64_t start = (int64_t)(b - p.block0[lo]) * IAF_OPT_TILE;
  const int64_t rem = T.numel - start;
  const int len = rem < IAF_OPT_TILE ? (int)rem : IAF_OPT_TILE;
  const int64_t s = T.offset + start;
  if (T.grad)
    eve_tile<true>(p, T.param + start, T.grad + start, p.mom1 + s, p.mom_max + s, p.delta + s, p.avg + s,
                   p.lookahead + s, len);
  else
    eve_tile<false>(p, T.param + start, nullptr, p.mom1 + s, p.mom_max + s, p.delta + s, p.avg + s, p.lookahead + s,
                    len);
}

// The launcher behind iaf_eve_step (iaf_capi.cu validates the arguments first).
static int iaf_eve_launch(const iaf_adamax_tensor_t* tensors_host, int n_tensors, float* mom1, float* mom_max,
                          float* delta, float* avg, float* lookahead, double lr, double beta1, double beta2,
                          double beta3, float grad_scale, void* stream, uint64_t* launches) {
  IafEveParams p;
  p.mom1 = mom1;
  p.mom_max = mom_max;
  p.delta = delta;
  p.avg = avg;
  p.lookahead = lookahead;
  p.grad_scale = grad_scale;
  // optim.py:125-146 with alpha = -lr (models.py:571): python float constants, cast to floatX
  p.c[0] = (float)(-lr);
  p.c[1] = (float)(1.0 - beta1);
  p.c[2] = (float)beta1;
  p.c[3] = (float)(1.0 - beta2);
  p.c[4] = 1e-8f;
  p.c[5] = (float)beta3;
  p.c[6] = (float)(1.0 - beta3);
  p.c[7] = (float)((1.0 - beta1) / beta1);

  cudaStream_t st = (cudaStream_t)stream;
  return iaf_opt_launch_chunks(p, tensors_host, n_tensors, launches, "iaf_eve_kernel", [&](int blocks) {
    IAF_LAUNCH(iaf_eve_kernel, blocks, IAF_OPT_THREADS, 0, st, p);
  });
}

namespace {
struct IafAdamaxRegister {
  IafAdamaxRegister() { iaf_adamax = IafAdamaxKernel{iaf_adamax_launch, iaf_eve_launch}; }
} iaf_adamax_register;
}  // namespace
