// Shared helpers for the pase_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <utility>
#include "../../include/pase_b200.h"

void pase_set_error(const char* fmt, ...);

#define PASE_CHECK_ARG(cond, ...)                     \
  do {                                                \
    if (!(cond)) {                                    \
      pase_set_error(__VA_ARGS__);                    \
      return PASE_ERR_ARG;                            \
    }                                                 \
  } while (0)

#define PASE_LAUNCH_CHECK(name)                                            \
  do {                                                                     \
    cudaError_t e__ = cudaGetLastError();                                  \
    if (e__ != cudaSuccess) {                                              \
      pase_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return (int)e__;                                                     \
    }                                                                      \
  } while (0)

static inline int pase_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

// ---- split-K weight gradients (splitk.cu) ----
// A split GEMM writes split z's partial tile t (128 x bn fp32, bn <= 128) at
// ws + (z * tiles + t) * 128 * bn; pase_splitk_reduce sums the splits in split order into C
// (C = sum, or C += sum when accumulating).  The workspace holds pase_splitk_ws_tiles() tiles
// of PASE_SPLITK_TILE floats, so a launch needs splits * tiles <= pase_splitk_ws_tiles().
// One workspace per device, shared by every split GEMM: calls must be ordered on one stream.
#define PASE_SPLITK_WAVES 4
#define PASE_SPLITK_TILE (128 * 128)
long pase_splitk_ws_tiles();
float* pase_splitk_workspace(cudaStream_t st, const char* who);
int pase_splitk_reduce(const float* ws, int splits, int tiles_j, int bn, long tiles, float* C,
                       long ldc, int I, int J, int accumulate, cudaStream_t st, const char* who);

// ---- programmatic dependent launch (PDL) ----
// Kernels launched through PASE_LAUNCH may be scheduled while the previous kernel of the stream
// is still draining (graph capture turns this into a programmatic edge): launch latency, block
// distribution and the kernel's own prologue overlap the predecessor's tail.  Contract: such a
// kernel executes pdl_wait() before its first access to global memory (the wait returns once
// every prerequisite grid has completed and flushed).
// Inside the CUDA-graph replay of the encoder step the attribute hides little launch latency,
// and the early trigger below lets the dependents' resident, waiting blocks get in the way of
// the running kernel, so it is OFF unless PASE_B200_PDL=1; with the attribute off pdl_wait()
// is a no-op.
static inline bool pase_pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PASE_B200_PDL");
    v = (e && atoi(e) == 1) ? 1 : 0;
  }
  return v == 1;
}
template <typename... KArgs, typename... Args>
static inline cudaError_t pase_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block,
                                          size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pase_pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}
#define PASE_LAUNCH(kern, grid, block, smem, st, ...) \
  pase_launch_pdl(kern, dim3(grid), dim3(block), (size_t)(smem), (cudaStream_t)(st), __VA_ARGS__)
// wait for the prerequisite grids, then let the NEXT kernel of the stream start its own
// launch / prologue (it waits for this grid's completion in turn)
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// reflect index for F.pad(mode='reflect'): t in [-padL, T+padR) -> [0,T)
__device__ __forceinline__ int reflect_idx(int t, int T) {
  if (t < 0) t = -t;
  if (t >= T) t = 2 * (T - 1) - t;
  return t;
}

// Packed variable-length row map of the *_gemm_nt_var entry points.  tab: 3n+1 ints, row0[0..n]
// (first GEMM row of each utterance, ascending; row0[n] = rows in use), then orow0[n] (first
// output row) and t_valid[n].  Row m of utterance i is its local row u = m - row0[i], stored at
// output row orow0[i] + u.  Returns false for rows past row0[n].
__device__ __forceinline__ bool var_row(const int* __restrict__ tab, int n, int m, int& orow,
                                        int& t_valid, int& u) {
  if (m >= __ldg(tab + n)) return false;
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(tab + mid) <= m) lo = mid;
    else hi = mid - 1;
  }
  u = m - __ldg(tab + lo);
  orow = __ldg(tab + n + 1 + lo) + u;
  t_valid = __ldg(tab + 2 * n + 1 + lo);
  return true;
}

// ---- storage formats of activation-sized tensors (C-ABI `*_fmt` / `*_bf16` arguments) ----
//   PASE_FMT_F32     fp32 (optionally with a tf32-residual twin for the 3xTF32 GEMM mode)
//   PASE_FMT_BF16    bf16
//   PASE_FMT_F16X2   fp16 pair x = hi + 2^-11 lo' (3xF16 GEMM mode), two arrays
#define PASE_FMT_F32 0
#define PASE_FMT_BF16 1
#define PASE_FMT_F16X2 2
#define PASE_F16_LO_MUL 2048.0f        // lo' = rn_f16((x - hi) * 2^11)

// 4 consecutive elements <-> float4 (fp32: 16-byte, bf16: 8-byte accesses)
__device__ __forceinline__ float4 ld4t(const float* p) {
  return *reinterpret_cast<const float4*>(p);
}
__device__ __forceinline__ float4 ld4t(const __nv_bfloat16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&u.x);
  const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&u.y);
  const float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
  return make_float4(fa.x, fa.y, fb.x, fb.y);
}
__device__ __forceinline__ void st4t(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4t(__nv_bfloat16* p, float4 v) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&a);
  u.y = *reinterpret_cast<const uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
// round-trip through the storage type (what a later reader of the stored value sees)
__device__ __forceinline__ float4 rt4t(const float*, float4 v) { return v; }
__device__ __forceinline__ float4 rt4t(const __nv_bfloat16*, float4 v) {
  return make_float4(__bfloat162float(__float2bfloat16_rn(v.x)),
                     __bfloat162float(__float2bfloat16_rn(v.y)),
                     __bfloat162float(__float2bfloat16_rn(v.z)),
                     __bfloat162float(__float2bfloat16_rn(v.w)));
}
// fp16 pair of the 3xF16 GEMM mode: hi = rn_f16(x), lo' = rn_f16((x - hi) * 2^11)
__device__ __forceinline__ void f16_split(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn((x - __half2float(hi)) * PASE_F16_LO_MUL);
}
__device__ __forceinline__ void st4_f16x2(__half* hi, __half* lo, float4 v) {
  __half h[4], l[4];
  f16_split(v.x, h[0], l[0]);
  f16_split(v.y, h[1], l[1]);
  f16_split(v.z, h[2], l[2]);
  f16_split(v.w, h[3], l[3]);
  *reinterpret_cast<uint2*>(hi) = *reinterpret_cast<const uint2*>(h);
  *reinterpret_cast<uint2*>(lo) = *reinterpret_cast<const uint2*>(l);
}
// lo = rn_tf32(x - trunc_tf32(x)): the part of x the tensor core drops when it reads x as tf32
__device__ __forceinline__ float tf32_residual(float x) {
  const float r = x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  uint32_t u = __float_as_uint(r);
  u += 0xFFFu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xFFFFE000u);
}
// Power-of-two scale that places values bounded by `bound` (> 0) below 2^14 in fp16 (3xF16
// gradient operands): s = 2^(14 - ceil(log2(bound))), clamped to a finite range; 1 for 0.
__device__ __forceinline__ float f16_grad_scale(float bound) {
  if (!(bound > 0.f) || !(bound < 3.0e38f)) return 1.f;
  int e;
  frexpf(bound, &e);                    // bound = m * 2^e, m in [0.5, 1)  ->  bound <= 2^e
  int k = 14 - e;
  k = k > 100 ? 100 : (k < -100 ? -100 : k);
  return ldexpf(1.f, k);
}
// max over non-negative floats through their bit patterns (order-preserving for x >= 0)
__device__ __forceinline__ void atomic_max_pos(float* addr, float v) {
  atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
