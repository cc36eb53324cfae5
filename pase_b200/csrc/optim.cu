// Flat-buffer Adam / RAdam: ONE launch updates every parameter of the model (encoder + all
// worker heads) with per-segment hyper-parameters and algorithm.  Replaces the 13 optimizer
// instances the reference steps one after the other (pase/models/WorkerScheduler/trainer.py:
// 86-143, worker_scheduler.py:66-73), and folds the 1/world gradient scale of the
// data-parallel all-reduce into the same pass.  Per segment:
//   Adam   torch.optim.Adam (amsgrad off, maximize off, L2 weight decay added to the gradient)
//   RAdam  the reference's RAdam (WorkerScheduler/radam.py): rectified step once rho >= 5,
//          un-normalised momentum step before, decoupled weight decay p += -(wd*lr)*p
#include "common.cuh"
#include <cstring>

namespace {

constexpr int SEG_MAX = 64;

struct AdamSeg {           // one row of the device segment table (6 x 8 bytes)
  long start, end;         // element range [start, end) of the flat buffers
  float lr, beta1, beta2, eps, weight_decay;
  float algorithm;         // 0: Adam, 1: RAdam
  long step_index;         // index into the device step-count vector
};

enum : int { UPD_ADAM = 0, UPD_RADAM_RECT = 1, UPD_RADAM_SGD = 2 };

struct SegConst {          // per-segment constants of one step, computed once per block
  float step_size;         // Adam: lr / (1 - beta1^t); RAdam: the fp64 step size, rounded
  float inv_sqrt_b2;       // Adam: 1 / sqrt(1 - beta2^t)
  float decay;             // RAdam: -(weight_decay * lr)
  int mode;                // UPD_*
};

// t = the segment's step count, already incremented for this update.  RAdam's rho is the
// difference of two numbers near 2/(1-beta2) (~2000 for beta2 = 0.999) that lands within
// 0.004 of the threshold 5 at steps 5 and 6: it and the step size are computed in fp64, as the
// reference computes them in Python floats.  The branch is chosen here, from the device step
// count, so a captured graph crosses rho = 5 by itself.
__device__ __forceinline__ SegConst seg_constants(const AdamSeg& sg, float t) {
  SegConst c;
  if (sg.algorithm == 0.f) {
    const float b1 = 1.f - powf(sg.beta1, t), b2 = 1.f - powf(sg.beta2, t);
    c.step_size = sg.lr / b1;
    c.inv_sqrt_b2 = rsqrtf(b2);
    c.decay = 0.f;
    c.mode = UPD_ADAM;
    return c;
  }
  const double td = (double)t, lr = (double)sg.lr, beta2 = (double)sg.beta2;
  const double b2t = pow(beta2, td);
  const double bias1 = 1.0 - pow((double)sg.beta1, td);
  const double rho_inf = 2.0 / (1.0 - beta2) - 1.0;
  const double rho = rho_inf - 2.0 * td * b2t / (1.0 - b2t);
  double step_size;
  if (rho >= 5.0) {
    step_size = lr * sqrt((1.0 - b2t) * (rho - 4.0) / (rho_inf - 4.0) * (rho - 2.0) / rho *
                          rho_inf / (rho_inf - 2.0)) / bias1;
    c.mode = UPD_RADAM_RECT;
  } else {
    step_size = lr / bias1;
    c.mode = UPD_RADAM_SGD;
  }
  c.step_size = (float)step_size;
  c.inv_sqrt_b2 = 0.f;
  c.decay = (float)(-((double)sg.weight_decay * lr));
  return c;
}

// One element of one segment: the arithmetic both kernels share.  g is the raw gradient,
// gscale its factor (grad_scale, or 1/world of the peers' sum).
__device__ __forceinline__ void seg_update(float& p, float& m, float& v, float g, float gscale,
                                           const AdamSeg& sg, const SegConst& c) {
  const float beta1 = sg.beta1, beta2 = sg.beta2, eps = sg.eps;
  if (c.mode == UPD_ADAM) {
    const float gg = g * gscale + sg.weight_decay * p;
    m = beta1 * m + (1.f - beta1) * gg;
    v = beta2 * v + (1.f - beta2) * gg * gg;
    const float denom = sqrtf(v) * c.inv_sqrt_b2 + eps;
    p -= c.step_size * m / denom;
    return;
  }
  // RAdam, in the order of the reference's tensor ops; decay is 0 when weight_decay is
  const float gg = g * gscale;
  m = beta1 * m + (1.f - beta1) * gg;
  v = beta2 * v + (1.f - beta2) * gg * gg;
  p = p + c.decay * p;
  if (c.mode == UPD_RADAM_RECT)
    p = p + (-c.step_size) * (m / (sqrtf(v) + eps));
  else
    p = p + (-c.step_size) * m;
}

__global__ void __launch_bounds__(256)
adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                 float* __restrict__ v, long n, const AdamSeg* __restrict__ segs, int nseg,
                 const float* __restrict__ steps, float grad_scale) {
  pdl_wait();
  __shared__ AdamSeg ss[SEG_MAX];
  __shared__ SegConst cs[SEG_MAX];
  for (int i = threadIdx.x; i < nseg; i += blockDim.x) {
    ss[i] = segs[i];
    cs[i] = seg_constants(ss[i], steps[ss[i].step_index]);
  }
  __syncthreads();
  const long stride = (long)gridDim.x * blockDim.x * 4;
  int s = 0;
  for (long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    while (s + 1 < nseg && i >= ss[s].end) ++s;
    // a float4 never straddles two segments when every segment starts at a multiple of 4
    // (the host pads); the scalar tail handles a ragged end
    const AdamSeg& sg = ss[s];
    const SegConst c = cs[s];
    const int cnt = (i + 3 < n) ? 4 : (int)(n - i);
    float pv[4], gv[4], mv[4], vv[4];
    if (cnt == 4) {
      const float4 P = *reinterpret_cast<const float4*>(p + i);
      const float4 G = *reinterpret_cast<const float4*>(g + i);
      const float4 M = *reinterpret_cast<const float4*>(m + i);
      const float4 V = *reinterpret_cast<const float4*>(v + i);
      pv[0] = P.x; pv[1] = P.y; pv[2] = P.z; pv[3] = P.w;
      gv[0] = G.x; gv[1] = G.y; gv[2] = G.z; gv[3] = G.w;
      mv[0] = M.x; mv[1] = M.y; mv[2] = M.z; mv[3] = M.w;
      vv[0] = V.x; vv[1] = V.y; vv[2] = V.z; vv[3] = V.w;
    } else {
      for (int k = 0; k < cnt; ++k) { pv[k] = p[i + k]; gv[k] = g[i + k]; mv[k] = m[i + k]; vv[k] = v[i + k]; }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k >= cnt) break;
      if (i + k >= sg.end) continue;                 // padding between segments: untouched
      seg_update(pv[k], mv[k], vv[k], gv[k], grad_scale, sg, c);
    }
    if (cnt == 4) {
      *reinterpret_cast<float4*>(p + i) = make_float4(pv[0], pv[1], pv[2], pv[3]);
      *reinterpret_cast<float4*>(m + i) = make_float4(mv[0], mv[1], mv[2], mv[3]);
      *reinterpret_cast<float4*>(v + i) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    } else {
      for (int k = 0; k < cnt; ++k) { p[i + k] = pv[k]; m[i + k] = mv[k]; v[i + k] = vv[k]; }
    }
  }
}

// ---- data parallelism fused into the update: reduce-scatter + Adam + all-gather ----
// Every rank's flat gradient / parameter buffers are mapped into every other rank's address
// space (CUDA IPC over NVLink / NVSwitch peer access).  Rank r owns the shard
// [lo_r, hi_r) of the flat index space.  ONE kernel per rank and step:
//   barrier A   my gradients are complete -> flag in every peer; wait for theirs
//   shard       g = mean_p grad_p[i] read straight from the peers' buffers (ld.cv), the
//               segment's update (seg_update) on the local (m, v, p) shard, the new parameter value stored into EVERY rank's
//               parameter buffer
//   barrier B   all my remote stores are performed -> flag in every peer; the LAST block
//               of the grid waits for the peers' flags before the kernel may complete (the
//               next forward reads parameters the peers wrote, and the next backward
//               overwrites gradients the peers read)
// No collective library call, no separate optimizer launch, nothing for the host to order: the
// step stays one CUDA graph.  NVLink traffic per rank and step: (W-1)/W of the gradient bytes
// in, the same out -- the reduce-scatter + all-gather volume of a ring, without its W-1 hops.
struct DpArgs {
  float* const* param_peers;       // [world] device pointers to every rank's flat parameters
  const float* const* grad_peers;  // [world]
  int* const* flag_peers;          // [world] each: int[2 * world]  (A flags | B flags)
  float* m;
  float* v;
  long n;
  const AdamSeg* segs;
  int nseg;
  const float* steps;
  int world, rank;
  int* epoch;                      // device scalar, advanced by this kernel
  unsigned* done;                  // device scalar, block counter of barrier B
};

__device__ __forceinline__ void st_flag_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_flag_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// spin until every rank's flag reached `want`; a peer that never arrives traps after ~20 s
__device__ __forceinline__ void wait_flags(const int* flags, int world, int want) {
  const long long t0 = clock64();
  for (int q = 0; q < world; ++q) {
    while (ld_flag_sys(flags + q) < want) {
      if (clock64() - t0 > 40000000000LL) __trap();
    }
  }
}

__global__ void __launch_bounds__(256)
adam_flat_dp_kernel(const DpArgs a) {
  __shared__ AdamSeg ss[SEG_MAX];
  __shared__ SegConst cs[SEG_MAX];
  __shared__ int s_last;
  const int W = a.world, R = a.rank;
  const int want = *reinterpret_cast<volatile int*>(a.epoch) + 1;
  for (int i = threadIdx.x; i < a.nseg; i += blockDim.x) {
    ss[i] = a.segs[i];
    cs[i] = seg_constants(ss[i], a.steps[ss[i].step_index]);
  }
  // ---- barrier A: the kernel is stream-ordered after backward, so my gradients are final
  if (blockIdx.x == 0 && threadIdx.x < W) {
    __threadfence_system();
    st_flag_sys(a.flag_peers[threadIdx.x] + R, want);
  }
  if (threadIdx.x == 0) wait_flags(a.flag_peers[R], W, want);
  __syncthreads();
  // ---- my shard: float4 granules [lo, hi)
  const long n4 = (a.n + 3) / 4;
  const long per = (n4 + W - 1) / W;
  const long lo = per * R * 4;
  long hi = per * (R + 1) * 4;
  if (hi > a.n) hi = a.n;
  const float inv_w = 1.f / (float)W;
  const long stride = (long)gridDim.x * blockDim.x * 4;
  int s = 0;
  for (long i = lo + ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < hi; i += stride) {
    while (s + 1 < a.nseg && i >= ss[s].end) ++s;
    const AdamSeg& sg = ss[s];
    const SegConst c = cs[s];
    // the flat buffers are padded to a multiple of 4 elements: whole float4 accesses
    float4 G = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = 0; q < W; ++q) {
      const float4 x = __ldcv(reinterpret_cast<const float4*>(a.grad_peers[q] + i));
      G.x += x.x; G.y += x.y; G.z += x.z; G.w += x.w;
    }
    const float4 P = *reinterpret_cast<const float4*>(a.param_peers[R] + i);
    const float4 M = *reinterpret_cast<const float4*>(a.m + i);
    const float4 V = *reinterpret_cast<const float4*>(a.v + i);
    float pv[4] = {P.x, P.y, P.z, P.w}, gv[4] = {G.x, G.y, G.z, G.w};
    float mv[4] = {M.x, M.y, M.z, M.w}, vv[4] = {V.x, V.y, V.z, V.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i + k >= sg.end) continue;                 // padding between segments: untouched
      seg_update(pv[k], mv[k], vv[k], gv[k], inv_w, sg, c);
    }
    const float4 Pn = make_float4(pv[0], pv[1], pv[2], pv[3]);
    *reinterpret_cast<float4*>(a.m + i) = make_float4(mv[0], mv[1], mv[2], mv[3]);
    *reinterpret_cast<float4*>(a.v + i) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    for (int q = 0; q < W; ++q) *reinterpret_cast<float4*>(a.param_peers[q] + i) = Pn;
  }
  // ---- barrier B
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(a.done, 1u);
    s_last = (prev == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (s_last) {
    if (threadIdx.x < W) {
      __threadfence_system();
      st_flag_sys(a.flag_peers[threadIdx.x] + W + R, want);
    }
    if (threadIdx.x == 0) {
      wait_flags(a.flag_peers[R] + W, W, want);
      *a.done = 0u;
      *reinterpret_cast<volatile int*>(a.epoch) = want;
      __threadfence();
    }
  }
}

}  // namespace

extern "C" {

int pase_adam_flat(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long n,
                   const long* seg_table, int nseg, const float* steps, float grad_scale,
                   void* stream) {
  PASE_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && seg_table && steps && n > 0,
                 "pase_adam_flat: null pointer / empty buffer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= SEG_MAX, "pase_adam_flat: nseg=%d (1..%d)", nseg, SEG_MAX);
  PASE_CHECK_ARG(aligned16(param) && aligned16(grad) && aligned16(exp_avg) && aligned16(exp_avg_sq),
                 "pase_adam_flat: buffers must be 16-byte aligned");
  static_assert(sizeof(AdamSeg) == 48, "segment row = 6 x 8 bytes");
  long blocks = (n / 4 + 255) / 256;
  const long cap = (long)pase_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  PASE_LAUNCH((adam_flat_kernel), (unsigned)blocks, 256, 0, (cudaStream_t)stream, 
      param, grad, exp_avg, exp_avg_sq, n, reinterpret_cast<const AdamSeg*>(seg_table), nseg, steps,
      grad_scale);
  PASE_LAUNCH_CHECK("pase_adam_flat");
  return PASE_OK;
}

int pase_adam_flat_dp(void* const* param_peers, void* const* grad_peers,
                      void* const* flag_peers, float* exp_avg, float* exp_avg_sq, long n,
                      const long* seg_table, int nseg, const float* steps, int world, int rank,
                      int* epoch, int* done, void* stream) {
  PASE_CHECK_ARG(param_peers && grad_peers && flag_peers && exp_avg && exp_avg_sq && seg_table &&
                     steps && epoch && done && n > 0,
                 "pase_adam_flat_dp: null pointer / empty buffer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= SEG_MAX, "pase_adam_flat_dp: nseg=%d (1..%d)", nseg, SEG_MAX);
  PASE_CHECK_ARG(world >= 1 && world <= 16 && rank >= 0 && rank < world && (n % 4) == 0,
                 "pase_adam_flat_dp: world=%d rank=%d n=%ld (n must be a multiple of 4)", world,
                 rank, n);
  PASE_CHECK_ARG(aligned16(exp_avg) && aligned16(exp_avg_sq),
                 "pase_adam_flat_dp: buffers must be 16-byte aligned");
  DpArgs a{reinterpret_cast<float* const*>(param_peers),
           reinterpret_cast<const float* const*>(grad_peers),
           reinterpret_cast<int* const*>(flag_peers), exp_avg, exp_avg_sq, n,
           reinterpret_cast<const AdamSeg*>(seg_table), nseg, steps, world, rank, epoch,
           reinterpret_cast<unsigned*>(done)};
  const long shard4 = ((n + 3) / 4 + world - 1) / world;
  long blocks = (shard4 + 255) / 256;
  // one wave of 8 x 256 threads per SM: every thread has its remote loads (NVLink latency
  // ~3 us) in flight at once instead of walking a long grid-stride loop.  (Blocks wait for
  // the PEERS in barrier A, never for each other, so more waves would also be correct.)
  const long cap = (long)pase_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  adam_flat_dp_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(a);
  PASE_LAUNCH_CHECK("pase_adam_flat_dp");
  return PASE_OK;
}

// ---- peer-mapped buffers (CUDA IPC) for pase_adam_flat_dp ----
// A dedicated cudaMalloc allocation per buffer: the IPC handle then names exactly this
// buffer (a caching-allocator block would export its whole segment at an unknown offset).
int pase_dp_alloc(long bytes, void** ptr_out, void* handle_out64) {
  PASE_CHECK_ARG(bytes > 0 && ptr_out && handle_out64, "pase_dp_alloc: bad args");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle = 64 bytes");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, (size_t)bytes);
  if (e == cudaSuccess) e = cudaMemset(p, 0, (size_t)bytes);
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle_out64), p);
  if (e != cudaSuccess) {
    pase_set_error("pase_dp_alloc(%ld bytes): %s", bytes, cudaGetErrorString(e));
    if (p) cudaFree(p);
    return (int)e;
  }
  *ptr_out = p;
  return PASE_OK;
}

// maps a peer process's buffer into the CURRENT device's address space (peer access over
// NVLink is enabled by the runtime as part of the open)
int pase_dp_open(const void* handle64, void** ptr_out) {
  PASE_CHECK_ARG(handle64 && ptr_out, "pase_dp_open: bad args");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    pase_set_error("pase_dp_open: %s", cudaGetErrorString(e));
    return (int)e;
  }
  *ptr_out = p;
  return PASE_OK;
}

int pase_dp_close(void* ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  if (e != cudaSuccess) {
    pase_set_error("pase_dp_close: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return PASE_OK;
}

int pase_dp_free(void* ptr) {
  cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) {
    pase_set_error("pase_dp_free: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return PASE_OK;
}

}  // extern "C"
