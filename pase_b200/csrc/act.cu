// Padding, BatchNorm (batch statistics), PReLU and dense-skip pooling kernels.
// All HBM-bound: channel-last float4 accesses, one pass per tensor.
#include "common.cuh"
#include "bn_stream.cuh"
#include <type_traits>

namespace {

constexpr int THREADS = 256;
// time steps per thread of the register-resident BatchNorm / PReLU kernels (measured 3.31 vs
// 3.42 ms/step against 4 steps per thread with 2-3 resident blocks per SM: loads in flight per
// thread matter more than occupancy here)
constexpr int RUN = 8;
// threads per block of the forward kernels, and blocks per SM their register budget must allow:
// 7 x 128 threads (72 registers) keep block 0's grid of 32 x 200 windows x 16 channel quads
// (800 blocks) resident in one wave on 132 SMs, where 3 x 256 threads (80 registers) left 4 of
// its 400 blocks to start only as the first ones finished.  The fp32 operand writer (with its
// optional tf32 residual) needs more than 72 and keeps 6 x 128, as does the packed form.
constexpr int FWD_THREADS = 128;
template <int DF>
constexpr int fwd_min_blocks() { return DF == PASE_FMT_F32 ? 6 : 7; }

// One utterance's reflect pad: dst[d0 + tau] = xn[reflect(tau - padL)] for tau < Tp.
// DF: operand format of the padded waveform (block 0's GEMM operand)
template <int DF>
__device__ __forceinline__ void reflect_pad_wave_utt(const float* __restrict__ xn, int T, int padL,
                                                     int Tp, void* __restrict__ dst_v,
                                                     void* __restrict__ dst_lo_v, long d0) {
  for (int tau = blockIdx.x * blockDim.x + threadIdx.x; tau < Tp; tau += gridDim.x * blockDim.x) {
    const float v = xn[reflect_idx(tau - padL, T)];
    const long o = d0 + tau;
    if constexpr (DF == PASE_FMT_F32) {
      reinterpret_cast<float*>(dst_v)[o] = v;
      if (dst_lo_v != nullptr) reinterpret_cast<float*>(dst_lo_v)[o] = tf32_residual(v);
    } else if constexpr (DF == PASE_FMT_BF16) {
      reinterpret_cast<__nv_bfloat16*>(dst_v)[o] = __float2bfloat16_rn(v);
    } else {
      __half h, l;
      f16_split(v, h, l);
      reinterpret_cast<__half*>(dst_v)[o] = h;
      reinterpret_cast<__half*>(dst_lo_v)[o] = l;
    }
  }
}

template <int DF>
__global__ void reflect_pad_wave_kernel(const float* __restrict__ x, void* __restrict__ dst_v,
                                        void* __restrict__ dst_lo_v, int T, int padL, int Tp,
                                        long pitch) {
  pdl_wait();
  const int n = blockIdx.y;
  reflect_pad_wave_utt<DF>(x + (long)n * T, T, padL, Tp, dst_v, dst_lo_v, (long)n * pitch);
}

// Packed variable-length form: blockIdx.y = utterance, tab row {x_off, T, dst_off}.
template <int DF>
__global__ void reflect_pad_wave_var_kernel(const float* __restrict__ x, const int* __restrict__ tab,
                                            void* __restrict__ dst_v, void* __restrict__ dst_lo_v,
                                            int padL, int padR) {
  pdl_wait();
  const int* r = tab + 3 * blockIdx.y;
  const int T = __ldg(r + 1);
  reflect_pad_wave_utt<DF>(x + __ldg(r), T, padL, T + padL + padR, dst_v, dst_lo_v, __ldg(r + 2));
}

// Calls f(std::integral_constant<int, DF>()) for the operand format fmt (checked by the caller).
template <typename F>
void with_fmt(int fmt, F f) {
  if (fmt == PASE_FMT_F32) f(std::integral_constant<int, PASE_FMT_F32>());
  else if (fmt == PASE_FMT_BF16) f(std::integral_constant<int, PASE_FMT_BF16>());
  else f(std::integral_constant<int, PASE_FMT_F16X2>());
}

__global__ void bn_finalize_kernel(const double* __restrict__ colsum,
                                   const double* __restrict__ colsumsq, int C, int fold,
                                   double count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* running_mean,
                                   float* running_var, float momentum, float eps, float* mean,
                                   float* invstd, float* scale, float* shift) {
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0, q = 0.0;
  for (int p = 0; p < fold; ++p) {
    s += colsum[p * C + c];
    q += colsumsq[p * C + c];
  }
  const double m = s / count;
  double var = q / count - m * m;
  if (var < 0.0) var = 0.0;
  const double is = 1.0 / sqrt(var + (double)eps);
  if (running_mean != nullptr) {
    const double unb = count > 1.0 ? var * count / (count - 1.0) : var;
    running_mean[c] = (float)((1.0 - momentum) * (double)running_mean[c] + momentum * m);
    running_var[c] = (float)((1.0 - momentum) * (double)running_var[c] + momentum * unb);
  }
  const double g = gamma ? (double)gamma[c] : 1.0;
  const double b = beta ? (double)beta[c] : 0.0;
  mean[c] = (float)m;
  invstd[c] = (float)is;
  scale[c] = (float)(g * is);
  shift[c] = (float)(b - m * g * is);
}

__global__ void bn_eval_affine_kernel(const float* __restrict__ rm, const float* __restrict__ rv,
                                      const float* __restrict__ gamma,
                                      const float* __restrict__ beta, int C, float eps,
                                      float* mean, float* invstd, float* scale, float* shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double is = 1.0 / sqrt((double)rv[c] + (double)eps);
  const double g = gamma ? (double)gamma[c] : 1.0;
  const double b = beta ? (double)beta[c] : 0.0;
  mean[c] = rm[c];
  invstd[c] = (float)is;
  scale[c] = (float)(g * is);
  shift[c] = (float)(b - (double)rm[c] * g * is);
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float prelu1(float u, float a) { return u > 0.f ? u : a * u; }

// Forward: a = PReLU(y*scale+shift) with reflect halo into the next layer's padded operand.
//   YT  storage type of y (float / bf16);  DF  operand format of dst:
//   PASE_FMT_F32 (+ optional tf32-residual twin dst_lo), PASE_FMT_BF16, PASE_FMT_F16X2
//   (dst = hi, dst_lo = lo').  The dense-skip pool accumulates the value the next layer
//   reads (i.e. after rounding to bf16 in the bf16 format).

// One activation of the channel quad at c, written at dst offset o; returns the value the next
// layer reads (the bf16-rounded one in the bf16 format), which is what the pool sums.
template <int DF>
__device__ __forceinline__ float4 bn_prelu_store(float4 v, float4 sc, float4 sh, float4 al,
                                                 void* __restrict__ dst_v,
                                                 void* __restrict__ dst_lo_v, long o) {
  float4 a;
  a.x = prelu1(fmaf(v.x, sc.x, sh.x), al.x);
  a.y = prelu1(fmaf(v.y, sc.y, sh.y), al.y);
  a.z = prelu1(fmaf(v.z, sc.z, sh.z), al.z);
  a.w = prelu1(fmaf(v.w, sc.w, sh.w), al.w);
  if constexpr (DF == PASE_FMT_F32) {
    st4(reinterpret_cast<float*>(dst_v) + o, a);
    if (dst_lo_v != nullptr)      // 3xTF32 residual of the operand just written
      st4(reinterpret_cast<float*>(dst_lo_v) + o,
          make_float4(tf32_residual(a.x), tf32_residual(a.y), tf32_residual(a.z),
                      tf32_residual(a.w)));
  } else if constexpr (DF == PASE_FMT_BF16) {
    __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dst_v) + o;
    st4t(d, a);
    a = rt4t(d, a);
  } else {
    st4_f16x2(reinterpret_cast<__half*>(dst_v) + o, reinterpret_cast<__half*>(dst_lo_v) + o, a);
  }
  return a;
}

// Runs of one sample's forward pass.  Without a pool (pool_d <= 0 or pool_T == 0) the padded
// output [0, Tp) is cut into runs of RUN time steps.  With one, the time steps are cut into
//   [0, padL)                        the left reflect halo, runs of RUN steps;
//   [padL, padL + pool_T * pool_d)   the pooled frames, runs of L = pool_d * ceil(RUN / pool_d)
//                                    steps: whole pooling windows only;
//   [padL + pool_T * pool_d, Tp)     the unpooled tail and the right halo, runs of RUN steps.
// Every window then lies inside one thread's run, and that thread sums it as it produces it.
struct FwdRuns {
  int nA, nB;             // runs of the left halo, of the pooled frames
  int wpr;                // pooling windows per pooled run
  int tail0;              // first time step of the runs after the pooled ones
  long total;             // all runs
};

__host__ __device__ __forceinline__ FwdRuns fwd_runs(int Tp, int padL, int pool_d, int pool_T) {
  FwdRuns r;
  if (pool_d > 0 && pool_T > 0) {
    r.nA = (padL + RUN - 1) / RUN;
    r.wpr = (RUN + pool_d - 1) / pool_d;
    r.nB = (pool_T + r.wpr - 1) / r.wpr;
    r.tail0 = padL + pool_T * pool_d;
  } else {
    r.nA = r.nB = r.wpr = r.tail0 = 0;
  }
  r.total = (long)r.nA + r.nB + (Tp - r.tail0 + RUN - 1) / RUN;
  return r;
}

// A pooled run: len time steps of the channel quad whose raw conv output starts at y, whole
// pooling windows of pd steps, streamed in chunks of RUN (RUN loads in flight, then compute and
// store).  Each activation is added to its window's sum in time order as it is produced; the
// window's mean goes to pp, the next window's to pp + p_rs.
template <typename YT, int DF>
__device__ __forceinline__ void bn_prelu_pooled_run(const YT* __restrict__ y, int C, int len,
                                                    int pd, float4 sc, float4 sh, float4 al,
                                                    void* __restrict__ dst_v,
                                                    void* __restrict__ dst_lo_v, long o, long d_rs,
                                                    float* __restrict__ pp, long p_rs) {
  float4 ps = make_float4(0.f, 0.f, 0.f, 0.f);
  int k = 0;                    // time steps of the current window summed so far
  for (int t0 = 0; t0 < len; t0 += RUN) {
    const int nvalid = min(RUN, len - t0);
    // straight-line loads (a step past the run re-reads the chunk's first row): no predicate, so
    // the chunk's registers never merge with the previous chunk's
    float4 vals[RUN];
#pragma unroll
    for (int i = 0; i < RUN; ++i) vals[i] = ld4t(y + (long)(t0 + (i < nvalid ? i : 0)) * C);
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      if (i >= nvalid) break;
      const float4 a = bn_prelu_store<DF>(vals[i], sc, sh, al, dst_v, dst_lo_v, o);
      o += d_rs;
      // round-to-nearest adds: the sum is never contracted into the PReLU multiply
      ps.x = __fadd_rn(ps.x, a.x); ps.y = __fadd_rn(ps.y, a.y);
      ps.z = __fadd_rn(ps.z, a.z); ps.w = __fadd_rn(ps.w, a.w);
      if (++k == pd) {
        const float inv_d = __frcp_rn((float)pd);     // = 1.f / pd, correctly rounded
        const float4 m = make_float4(ps.x * inv_d, ps.y * inv_d, ps.z * inv_d, ps.w * inv_d);
        // one 16-byte reduction per window where the quad is aligned (always in the uniform
        // launch; a packed table's pool_off need not be a multiple of 4)
        if ((reinterpret_cast<uintptr_t>(pp) & 15u) == 0) {
          atomicAdd(reinterpret_cast<float4*>(pp), m);
        } else {
          atomicAdd(pp + 0, m.x);
          atomicAdd(pp + 1, m.y);
          atomicAdd(pp + 2, m.z);
          atomicAdd(pp + 3, m.w);
        }
        pp += p_rs;
        ps = make_float4(0.f, 0.f, 0.f, 0.f);
        k = 0;
      }
    }
  }
}

// One sample: yn its raw conv output, dst / pool offsets d_base / p_base; thread idx owns the
// channel quad idx % (C/4) over run idx / (C/4) of fwd_runs.  A pooled run sums each of its
// windows in time order as it produces it (bn_prelu_pooled_run), so each window mean has one
// writer and comes out the same on every run.
template <typename YT, int DF>
__device__ __forceinline__ void bn_prelu_pad_fwd_sample(
    const YT* __restrict__ yn, long idx, int T, int C, const float* __restrict__ scale,
    const float* __restrict__ shift, const float* __restrict__ alpha, void* __restrict__ dst_v,
    long d_base, long d_rs, int padL, int Tp, float* __restrict__ pool, long p_base, long p_rs,
    int pool_d, int pool_T, void* __restrict__ dst_lo_v) {
  const int C4 = C >> 2;
  const int q = (int)(idx % C4);
  const long run = idx / C4;
  const FwdRuns R = fwd_runs(Tp, padL, pool_d, pool_T);
  if (run >= R.total) return;
  const int c = q * 4;
  const float4 sc = ld4(scale + c), sh = ld4(shift + c), al = ld4(alpha + c);
  if (run >= R.nA && run < R.nA + R.nB) {
    const int w0 = (int)(run - R.nA) * R.wpr;      // first window, first frame w0 * pool_d
    const int tr0 = w0 * pool_d;
    bn_prelu_pooled_run<YT, DF>(yn + (long)tr0 * C + c, C,
                                min(R.wpr, pool_T - w0) * pool_d, pool_d, sc, sh, al, dst_v,
                                dst_lo_v, d_base + (long)(padL + tr0) * d_rs + c, d_rs,
                                pool + p_base + (long)w0 * p_rs + c, p_rs);
    return;
  }
  // RUN padded time steps from tau0 (fewer at the end of their range): the left halo, the
  // unpooled tail and right halo, or any run of a launch without a pool
  const int tau0 = run < R.nA ? (int)run * RUN : R.tail0 + (int)(run - R.nA - R.nB) * RUN;
  const int tend = run < R.nA ? padL : Tp;
  const int nvalid = min(RUN, tend - tau0);
  float4 vals[RUN];
#pragma unroll
  for (int i = 0; i < RUN; ++i)
    if (i < nvalid) vals[i] = ld4t(yn + (long)reflect_idx(tau0 + i - padL, T) * C + c);
#pragma unroll
  for (int i = 0; i < RUN; ++i) {
    if (i >= nvalid) break;
    bn_prelu_store<DF>(vals[i], sc, sh, al, dst_v, dst_lo_v, d_base + (long)(tau0 + i) * d_rs + c);
  }
}

template <typename YT, int DF>
__global__ void __launch_bounds__(FWD_THREADS, fwd_min_blocks<DF>())
bn_prelu_pad_fwd_kernel(const YT* __restrict__ y, long y_ss, int T, int C,
                        const float* __restrict__ scale, const float* __restrict__ shift,
                        const float* __restrict__ alpha, void* __restrict__ dst_v, long d_ss,
                        long d_rs, int padL, int Tp, float* __restrict__ pool, long p_ss,
                        long p_rs, int pool_d, int pool_T, void* __restrict__ dst_lo_v) {
  pdl_wait();
  const int n = blockIdx.y;
  bn_prelu_pad_fwd_sample<YT, DF>(y + (long)n * y_ss,
                                  (long)blockIdx.x * blockDim.x + threadIdx.x, T, C, scale,
                                  shift, alpha, dst_v, (long)n * d_ss, d_rs, padL, Tp, pool,
                                  (long)n * p_ss, p_rs, pool_d, pool_T, dst_lo_v);
}

// Packed variable-length form: blockIdx.y = utterance, tab row {T, y_off, dst_off, pool_off,
// pool_d, pool_T} (elements).  sep != 0: the row ahead of each utterance's output (dst_off -
// d_rs, C elements) is written zero (the QRNN input's x_{-1} row).
template <typename YT, int DF>
__global__ void __launch_bounds__(FWD_THREADS, 6)   // the sep row and the table: 80 registers
bn_prelu_pad_fwd_var_kernel(const YT* __restrict__ y, const int* __restrict__ tab, int C,
                            const float* __restrict__ scale, const float* __restrict__ shift,
                            const float* __restrict__ alpha, void* __restrict__ dst_v, long d_rs,
                            int padL, int padR, float* __restrict__ pool, long p_rs, int sep,
                            void* __restrict__ dst_lo_v) {
  pdl_wait();
  const int* r = tab + 6 * blockIdx.y;
  const int T = __ldg(r), pool_d = pool != nullptr ? __ldg(r + 4) : 0;
  const long d_base = __ldg(r + 2);
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (sep && idx < (C >> 2)) {
    const long o = d_base - d_rs + 4 * idx;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (DF == PASE_FMT_F32) {
      st4(reinterpret_cast<float*>(dst_v) + o, z);
      if (dst_lo_v != nullptr) st4(reinterpret_cast<float*>(dst_lo_v) + o, z);
    } else if constexpr (DF == PASE_FMT_BF16) {
      st4t(reinterpret_cast<__nv_bfloat16*>(dst_v) + o, z);
    } else {
      st4_f16x2(reinterpret_cast<__half*>(dst_v) + o, reinterpret_cast<__half*>(dst_lo_v) + o, z);
    }
  }
  bn_prelu_pad_fwd_sample<YT, DF>(y + __ldg(r + 1), idx, T, C, scale, shift, alpha, dst_v,
                                  d_base, d_rs, padL, T + padL + padR, pool, __ldg(r + 3),
                                  p_rs, pool_d, __ldg(r + 5), dst_lo_v);
}

// ---- backward pass 1: du + reductions ----
// (BwdSrc: bn_stream.cuh)

// The gradient reaching this block's output for one run of RUN time steps (t0 ..) of the
// channel quad at c: source A (the next layer's padded input gradient, reflect halo folded
// back at the two sequence ends), the optional shifted source B (QRNN) and the broadcast of
// the mean-pooled dense-skip gradient.  Straight-line loads first (no branch between a load
// and the next one, so all DRAM requests of the run are in flight together).
template <typename GT>
__device__ __forceinline__ void load_grad_run(const BwdSrc& s, int n, int T, long t0, int nvalid,
                                              int c, float4 (&gs)[RUN]) {
  const GT* an = reinterpret_cast<const GT*>(s.A) + (long)n * s.a_ss + c;
#pragma unroll
  for (int i = 0; i < RUN; ++i) {
    const int t = (int)t0 + (i < nvalid ? i : 0);
    gs[i] = ld4t(an + (long)(t + s.padL) * s.a_rs);
  }
  if (s.P != nullptr && s.pool_d > 0) {       // mean-pooled dense-skip gradient (broadcast)
    const int pool_len = s.pool_T * s.pool_d;
    const float inv_d = 1.f / (float)s.pool_d;
    const float* pn = s.P + (long)n * s.p_ss + c;
    float4 pv[RUN];
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      const int t = (int)t0 + (i < nvalid ? i : 0);
      const int tw = t < pool_len ? t / s.pool_d : 0;
      pv[i] = ld4(pn + (long)tw * s.p_rs);
    }
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      const int t = (int)t0 + i;
      const float w = (t < pool_len) ? inv_d : 0.f;
      gs[i].x += pv[i].x * w; gs[i].y += pv[i].y * w;
      gs[i].z += pv[i].z * w; gs[i].w += pv[i].w * w;
    }
  }
  // rare: reflect-pad fold-back at the two sequence ends, second shifted source (QRNN)
  const bool edge = (s.padL > 0 && t0 <= s.padL) || (s.padR > 0 && t0 + RUN >= T - 1 - s.padR);
  if (edge || s.B != nullptr) {
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      if (i >= nvalid) break;
      const int t = (int)t0 + i;
      float4 g = gs[i];
      auto add4 = [&](float4 v) { g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w; };
      if (s.padL > 0 && t >= 1 && t <= s.padL) add4(ld4t(an + (long)(s.padL - t) * s.a_rs));
      if (s.padR > 0 && t <= T - 2 && t >= T - 1 - s.padR)
        add4(ld4t(an + (long)(s.padL + 2 * (T - 1) - t) * s.a_rs));
      if (s.B) {
        const int tb = t + s.b_shift;
        if (tb >= 0 && tb < T) add4(ld4(s.B + (long)n * s.b_ss + (long)tb * s.b_rs + c));
      }
      gs[i] = g;
    }
  }
}

// YT: storage type of y and of du (dst); GT: storage type of the gradient source A (the
// next layer's input gradient as its dgrad GEMM wrote it).  amax (optional, float[2]):
// running maxima of |du| and |xhat| (bit-pattern atomicMax), from which pass 2 derives the
// power-of-two scale of the fp16 gradient operand (3xF16 mode).
template <typename YT, typename GT>
__global__ void __launch_bounds__(THREADS, 1)
bn_prelu_bwd_reduce_kernel(const YT* __restrict__ y, long y_ss, int T, int C,
                           const float* __restrict__ mean, const float* __restrict__ invstd,
                           const float* __restrict__ scale, const float* __restrict__ shift,
                           const float* __restrict__ alpha, BwdSrc s, YT* __restrict__ dst,
                           long d_ss, double* __restrict__ S1, double* __restrict__ S2,
                           double* __restrict__ dalpha, float* __restrict__ amax) {
  // block sums [3][C] in fp64: the order of the threads' additions then only moves bits below
  // fp32 precision (run-to-run identical statistics); [2] maxima in fp32 after them
  extern __shared__ double red[];
  float* redm = reinterpret_cast<float*>(red + 3 * C);
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) red[i] = 0.0;
  if (threadIdx.x < 2) redm[threadIdx.x] = 0.f;
  __syncthreads();
  const int C4 = C >> 2;
  const int n = blockIdx.y;
  // grid-stride over runs (the host only caps the grid when the stride keeps each thread on
  // the same channel quad): fewer blocks -> far fewer same-address fp64 atomics at the end
  const long idx0 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long nthreads = (long)C4 * ((T + RUN - 1) / RUN);
  const int q = (int)(idx0 % C4);
  const int c = q * 4;
  float a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0}, a3[4] = {0, 0, 0, 0};
  float mx_du = 0.f, mx_xh = 0.f;
  const float4 sc = ld4(scale + c), sh = ld4(shift + c), al = ld4(alpha + c);
  const float4 mu = ld4(mean + c), is = ld4(invstd + c);
  const YT* yn = y + (long)n * y_ss;
  YT* dn = dst ? dst + (long)n * d_ss : nullptr;
  for (long idx = idx0; idx < nthreads; idx += (long)gridDim.x * blockDim.x) {
    const long t0 = (idx / C4) * RUN;
    const int nvalid = (T - (int)t0) < RUN ? (T - (int)t0) : RUN;
    float4 gs[RUN], ys[RUN];
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      const int t = (int)t0 + (i < nvalid ? i : 0);
      ys[i] = ld4t(yn + (long)t * C + c);
    }
    load_grad_run<GT>(s, n, T, t0, nvalid, c, gs);
    const float scv[4] = {sc.x, sc.y, sc.z, sc.w}, shv[4] = {sh.x, sh.y, sh.z, sh.w};
    const float alv[4] = {al.x, al.y, al.z, al.w};
    const float muv[4] = {mu.x, mu.y, mu.z, mu.w}, isv[4] = {is.x, is.y, is.z, is.w};
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      if (i >= nvalid) break;
      const int t = (int)t0 + i;
      const float gg[4] = {gs[i].x, gs[i].y, gs[i].z, gs[i].w};
      const float vv[4] = {ys[i].x, ys[i].y, ys[i].z, ys[i].w};
      float du[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float u = fmaf(vv[k], scv[k], shv[k]);
        const bool pos = u > 0.f;
        du[k] = pos ? gg[k] : alv[k] * gg[k];
        a3[k] += pos ? 0.f : u * gg[k];
        const float xh = (vv[k] - muv[k]) * isv[k];
        a1[k] += du[k];
        a2[k] += du[k] * xh;
        mx_du = fmaxf(mx_du, fabsf(du[k]));
        mx_xh = fmaxf(mx_xh, fabsf(xh));
      }
      if (dn != nullptr) st4t(dn + (long)t * C + c, make_float4(du[0], du[1], du[2], du[3]));
    }
  }
  // lanes that own the same channel quad (C/4 < 32, power of two) combine before the
  // shared-memory atomics; every lane of the warp takes part (idle lanes contribute zeros)
  const bool pre = (C4 < 32) && ((C4 & (C4 - 1)) == 0) && ((blockDim.x % C4) == 0);
  if (pre) {
    for (int off = 16; off >= C4; off >>= 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        a1[k] += __shfl_xor_sync(0xffffffffu, a1[k], off);
        a2[k] += __shfl_xor_sync(0xffffffffu, a2[k], off);
        a3[k] += __shfl_xor_sync(0xffffffffu, a3[k], off);
      }
    }
  }
  if ((pre && (threadIdx.x & 31) < C4) || (!pre && idx0 < nthreads)) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      atomicAdd(&red[0 * C + c + k], (double)a1[k]);
      atomicAdd(&red[1 * C + c + k], (double)a2[k]);
      atomicAdd(&red[2 * C + c + k], (double)a3[k]);
    }
  }
  if (amax != nullptr) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      mx_du = fmaxf(mx_du, __shfl_xor_sync(0xffffffffu, mx_du, off));
      mx_xh = fmaxf(mx_xh, __shfl_xor_sync(0xffffffffu, mx_xh, off));
    }
    if ((threadIdx.x & 31) == 0) {
      atomic_max_pos(&redm[0], mx_du);
      atomic_max_pos(&redm[1], mx_xh);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    atomicAdd(S1 + i, red[0 * C + i]);
    atomicAdd(S2 + i, red[1 * C + i]);
    atomicAdd(dalpha + i, red[2 * C + i]);
  }
  if (amax != nullptr && threadIdx.x == 0) {
    atomic_max_pos(amax, redm[0]);
    atomic_max_pos(amax + 1, redm[1]);
  }
}

// Backward pass 2: dy = gamma*invstd*(du - S1/M - xhat*S2/M), du read from `du` (may alias
// dst), dy written as the NEXT GEMMs' A operand in format DF.  PASE_FMT_F16X2: dy is scaled
// by the power of two derived from the bound
//     |dy| <= max_c |gamma_c invstd_c| (max|du| + |S1_c/M| + max|xhat| |S2_c/M|)
// (amax from pass 1), every block computes the same scale; block (0,0) publishes
// scale_out = {1/s, s} for the consuming GEMMs (alpha_dev).
template <typename YT, int DF>
__global__ void __launch_bounds__(THREADS, 2)
bn_prelu_bwd_apply_kernel(const YT* __restrict__ y, long y_ss, int T, int C,
                          const float* __restrict__ mean, const float* __restrict__ invstd,
                          const float* __restrict__ gamma, const double* __restrict__ S1,
                          const double* __restrict__ S2, double inv_count,
                          const YT* du, void* dst_v, long d_ss,
                          double* __restrict__ dbias, void* dst_lo_v,
                          const float* __restrict__ amax, float* __restrict__ scale_out) {
  extern __shared__ double red[];     // [C] fp64 sums (see pass 1), then [1] fp32 maximum
  float* redm = reinterpret_cast<float*>(red + C);
  for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.0;
  if (threadIdx.x == 0) redm[0] = 0.f;
  __syncthreads();
  float gs_scale = 1.f;
  if constexpr (DF == PASE_FMT_F16X2) {
    const float mdu = amax[0], mxh = amax[1];
    float b = 0.f;
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      const float gi = fabsf((gamma ? gamma[i] : 1.f) * invstd[i]);
      const float m1 = fabsf((float)(S1[i] * inv_count)), m2 = fabsf((float)(S2[i] * inv_count));
      b = fmaxf(b, gi * (mdu + m1 + mxh * m2));
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, off));
    if ((threadIdx.x & 31) == 0) atomic_max_pos(&redm[0], b);
    __syncthreads();
    gs_scale = f16_grad_scale(redm[0] * 1.0001f);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
      scale_out[0] = 1.f / gs_scale;
      scale_out[1] = gs_scale;
    }
  }
  const int C4 = C >> 2;
  const int n = blockIdx.y;
  const long idx0 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long nthreads = (long)C4 * ((T + RUN - 1) / RUN);
  const int q = (int)(idx0 % C4);
  const int c = q * 4;
  float acc[4] = {0, 0, 0, 0};
  if (idx0 < nthreads) {
    float m1[4], m2[4], gi[4], muv[4], isv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      m1[k] = (float)(S1[c + k] * inv_count);
      m2[k] = (float)(S2[c + k] * inv_count);
      muv[k] = mean[c + k];
      isv[k] = invstd[c + k];
      gi[k] = (gamma ? gamma[c + k] : 1.f) * isv[k];
    }
    const YT* yn = y + (long)n * y_ss;
    const YT* un = du + (long)n * d_ss;
    for (long idx = idx0; idx < nthreads; idx += (long)gridDim.x * blockDim.x) {
      const long t0 = (idx / C4) * RUN;
      const int nvalid = (T - (int)t0) < RUN ? (T - (int)t0) : RUN;
      float4 vs[RUN], ds[RUN];
#pragma unroll
      for (int i = 0; i < RUN; ++i)
        if (i < nvalid) {
          vs[i] = ld4t(yn + (long)((int)t0 + i) * C + c);
          ds[i] = ld4t(un + (long)((int)t0 + i) * C + c);
        }
#pragma unroll
      for (int i = 0; i < RUN; ++i) {
        if (i >= nvalid) break;
        const int t = (int)t0 + i;
        const float vv[4] = {vs[i].x, vs[i].y, vs[i].z, vs[i].w};
        const float dd[4] = {ds[i].x, ds[i].y, ds[i].z, ds[i].w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float xh = (vv[k] - muv[k]) * isv[k];
          o[k] = gi[k] * (dd[k] - m1[k] - xh * m2[k]);
          acc[k] += o[k];
        }
        const long off = (long)n * d_ss + (long)t * C + c;
        if constexpr (DF == PASE_FMT_F32) {
          st4(reinterpret_cast<float*>(dst_v) + off, make_float4(o[0], o[1], o[2], o[3]));
          if (dst_lo_v != nullptr)
            st4(reinterpret_cast<float*>(dst_lo_v) + off,
                make_float4(tf32_residual(o[0]), tf32_residual(o[1]), tf32_residual(o[2]),
                            tf32_residual(o[3])));
        } else if constexpr (DF == PASE_FMT_BF16) {
          st4t(reinterpret_cast<__nv_bfloat16*>(dst_v) + off, make_float4(o[0], o[1], o[2], o[3]));
        } else {
          st4_f16x2(reinterpret_cast<__half*>(dst_v) + off,
                    reinterpret_cast<__half*>(dst_lo_v) + off,
                    make_float4(o[0] * gs_scale, o[1] * gs_scale, o[2] * gs_scale,
                                o[3] * gs_scale));
        }
      }
    }
    if (dbias) {
#pragma unroll
      for (int k = 0; k < 4; ++k) atomicAdd(&red[c + k], (double)acc[k]);
    }
  }
  if (dbias) {
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(dbias + i, red[i]);
  }
}

// Backward pass 2 without a stored du: du = PReLU'(u) g is recomputed from the gradient
// sources (same arithmetic as pass 1, so the sums S1 / S2 it is centred with are exactly its
// own) -- pass 1 then writes nothing but its 3C sums, and the du tensor (one write + one read
// of the layer's activation size) disappears from the step.
template <typename YT, typename GT, int DF>
__global__ void __launch_bounds__(THREADS, 1)
bn_prelu_bwd_apply_src_kernel(const YT* __restrict__ y, long y_ss, int T, int C,
                              const float* __restrict__ mean, const float* __restrict__ invstd,
                              const float* __restrict__ gamma, const float* __restrict__ scale,
                              const float* __restrict__ shift, const float* __restrict__ alpha,
                              const double* __restrict__ S1, const double* __restrict__ S2,
                              double inv_count, BwdSrc s, void* dst_v, long d_ss,
                              double* __restrict__ dbias, void* dst_lo_v,
                              const float* __restrict__ amax, float* __restrict__ scale_out) {
  extern __shared__ double red[];     // [C] fp64 sums (see pass 1), then [1] fp32 maximum
  float* redm = reinterpret_cast<float*>(red + C);
  for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.0;
  if (threadIdx.x == 0) redm[0] = 0.f;
  __syncthreads();
  float gs_scale = 1.f;
  if constexpr (DF == PASE_FMT_F16X2) {
    const float mdu = amax[0], mxh = amax[1];
    float b = 0.f;
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      const float gi = fabsf((gamma ? gamma[i] : 1.f) * invstd[i]);
      const float m1 = fabsf((float)(S1[i] * inv_count)), m2 = fabsf((float)(S2[i] * inv_count));
      b = fmaxf(b, gi * (mdu + m1 + mxh * m2));
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, off));
    if ((threadIdx.x & 31) == 0) atomic_max_pos(&redm[0], b);
    __syncthreads();
    gs_scale = f16_grad_scale(redm[0] * 1.0001f);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
      scale_out[0] = 1.f / gs_scale;
      scale_out[1] = gs_scale;
    }
  }
  const int C4 = C >> 2;
  const int n = blockIdx.y;
  const long idx0 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long nthreads = (long)C4 * ((T + RUN - 1) / RUN);
  const int q = (int)(idx0 % C4);
  const int c = q * 4;
  float acc[4] = {0, 0, 0, 0};
  if (idx0 < nthreads) {
    float m1[4], m2[4], gi[4], muv[4], isv[4], scv[4], shv[4], alv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      m1[k] = (float)(S1[c + k] * inv_count);
      m2[k] = (float)(S2[c + k] * inv_count);
      muv[k] = mean[c + k];
      isv[k] = invstd[c + k];
      gi[k] = (gamma ? gamma[c + k] : 1.f) * isv[k];
      scv[k] = scale[c + k];
      shv[k] = shift[c + k];
      alv[k] = alpha[c + k];
    }
    const YT* yn = y + (long)n * y_ss;
    for (long idx = idx0; idx < nthreads; idx += (long)gridDim.x * blockDim.x) {
      const long t0 = (idx / C4) * RUN;
      const int nvalid = (T - (int)t0) < RUN ? (T - (int)t0) : RUN;
      float4 vs[RUN], gs[RUN];
#pragma unroll
      for (int i = 0; i < RUN; ++i) {
        const int t = (int)t0 + (i < nvalid ? i : 0);
        vs[i] = ld4t(yn + (long)t * C + c);
      }
      load_grad_run<GT>(s, n, T, t0, nvalid, c, gs);
#pragma unroll
      for (int i = 0; i < RUN; ++i) {
        if (i >= nvalid) break;
        const int t = (int)t0 + i;
        const float vv[4] = {vs[i].x, vs[i].y, vs[i].z, vs[i].w};
        const float gg[4] = {gs[i].x, gs[i].y, gs[i].z, gs[i].w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float u = fmaf(vv[k], scv[k], shv[k]);
          const float du = u > 0.f ? gg[k] : alv[k] * gg[k];
          const float xh = (vv[k] - muv[k]) * isv[k];
          o[k] = gi[k] * (du - m1[k] - xh * m2[k]);
          acc[k] += o[k];
        }
        const long off = (long)n * d_ss + (long)t * C + c;
        if constexpr (DF == PASE_FMT_F32) {
          st4(reinterpret_cast<float*>(dst_v) + off, make_float4(o[0], o[1], o[2], o[3]));
          if (dst_lo_v != nullptr)
            st4(reinterpret_cast<float*>(dst_lo_v) + off,
                make_float4(tf32_residual(o[0]), tf32_residual(o[1]), tf32_residual(o[2]),
                            tf32_residual(o[3])));
        } else if constexpr (DF == PASE_FMT_BF16) {
          st4t(reinterpret_cast<__nv_bfloat16*>(dst_v) + off, make_float4(o[0], o[1], o[2], o[3]));
        } else {
          st4_f16x2(reinterpret_cast<__half*>(dst_v) + off,
                    reinterpret_cast<__half*>(dst_lo_v) + off,
                    make_float4(o[0] * gs_scale, o[1] * gs_scale, o[2] * gs_scale,
                                o[3] * gs_scale));
        }
      }
    }
    if (dbias) {
#pragma unroll
      for (int k = 0; k < 4; ++k) atomicAdd(&red[c + k], (double)acc[k]);
    }
  }
  if (dbias) {
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(dbias + i, red[i]);
  }
}

// ---- packed variable-length backward (eval BatchNorm; pase_bn_prelu_bwd_*_var) ----
// Table row (ints) of utterance blockIdx.y: {T, y_off, a_off, b_off, pool_off, pool_d, pool_T,
// d_off, d_span}.  The gradient sources of one utterance are those of a B=1 call at the row's
// offsets, so load_grad_run (n = 0) gives the uniform kernels' sums in their order.
constexpr int BWD_ROW = 9;

template <typename GT>
__device__ __forceinline__ BwdSrc var_src(const int* r, const void* A, long a_rs, int padL,
                                          int padR, const float* B, long b_rs, int b_shift,
                                          const float* pool, long p_rs) {
  BwdSrc s;
  s.A = reinterpret_cast<const GT*>(A) + __ldg(r + 2); s.a_ss = 0; s.a_rs = a_rs;
  s.padL = padL; s.padR = padR;
  s.B = B ? B + __ldg(r + 3) : nullptr; s.b_ss = 0; s.b_rs = b_rs; s.b_shift = b_shift;
  s.P = pool ? pool + __ldg(r + 4) : nullptr; s.p_ss = 0; s.p_rs = p_rs;
  s.pool_d = pool ? __ldg(r + 5) : 0; s.pool_T = __ldg(r + 6);
  return s;
}

// pass 1 of pase_bn_prelu_bwd_reduce for every utterance: S1, S2, dalpha and the maxima
template <typename YT, typename GT>
__global__ void __launch_bounds__(THREADS)
bn_prelu_bwd_reduce_var_kernel(const YT* __restrict__ y, const int* __restrict__ tab, int C,
                               const float* __restrict__ mean, const float* __restrict__ invstd,
                               const float* __restrict__ scale, const float* __restrict__ shift,
                               const float* __restrict__ alpha, const void* A, long a_rs,
                               int padL, int padR, const float* B, long b_rs, int b_shift,
                               const float* pool, long p_rs, double* __restrict__ S1,
                               double* __restrict__ S2, double* __restrict__ dalpha,
                               float* __restrict__ amax) {
  pdl_wait();
  extern __shared__ double red[];
  float* redm = reinterpret_cast<float*>(red + 3 * C);
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) red[i] = 0.0;
  if (threadIdx.x < 2) redm[threadIdx.x] = 0.f;
  __syncthreads();
  const int* r = tab + BWD_ROW * blockIdx.y;
  const int T = __ldg(r);
  const BwdSrc s = var_src<GT>(r, A, a_rs, padL, padR, B, b_rs, b_shift, pool, p_rs);
  const int C4 = C >> 2;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long nthreads = (long)C4 * ((T + RUN - 1) / RUN);
  const int c = (int)(idx % C4) * 4;
  float a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0}, a3[4] = {0, 0, 0, 0};
  float mx_du = 0.f, mx_xh = 0.f;
  if (idx < nthreads) {
    const YT* yn = y + __ldg(r + 1);
    const long t0 = (idx / C4) * RUN;
    const int nvalid = (T - (int)t0) < RUN ? (T - (int)t0) : RUN;
    float4 gs[RUN], ys[RUN];
#pragma unroll
    for (int i = 0; i < RUN; ++i) ys[i] = ld4t(yn + (long)((int)t0 + (i < nvalid ? i : 0)) * C + c);
    load_grad_run<GT>(s, 0, T, t0, nvalid, c, gs);
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      if (i >= nvalid) break;
      const float gg[4] = {gs[i].x, gs[i].y, gs[i].z, gs[i].w};
      const float vv[4] = {ys[i].x, ys[i].y, ys[i].z, ys[i].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float u = fmaf(vv[k], scale[c + k], shift[c + k]);
        const bool pos = u > 0.f;
        const float du = pos ? gg[k] : alpha[c + k] * gg[k];
        a3[k] += pos ? 0.f : u * gg[k];
        const float xh = (vv[k] - mean[c + k]) * invstd[c + k];
        a1[k] += du;
        a2[k] += du * xh;
        mx_du = fmaxf(mx_du, fabsf(du));
        mx_xh = fmaxf(mx_xh, fabsf(xh));
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      atomicAdd(&red[0 * C + c + k], (double)a1[k]);
      atomicAdd(&red[1 * C + c + k], (double)a2[k]);
      atomicAdd(&red[2 * C + c + k], (double)a3[k]);
    }
  }
  if (amax != nullptr) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      mx_du = fmaxf(mx_du, __shfl_xor_sync(0xffffffffu, mx_du, off));
      mx_xh = fmaxf(mx_xh, __shfl_xor_sync(0xffffffffu, mx_xh, off));
    }
    if ((threadIdx.x & 31) == 0) {
      atomic_max_pos(&redm[0], mx_du);
      atomic_max_pos(&redm[1], mx_xh);
    }
  }
  __syncthreads();
  if ((long)blockIdx.x * blockDim.x < nthreads) {
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      atomicAdd(S1 + i, red[0 * C + i]);
      atomicAdd(S2 + i, red[1 * C + i]);
      atomicAdd(dalpha + i, red[2 * C + i]);
    }
  }
  if (amax != nullptr && threadIdx.x == 0) {
    atomic_max_pos(amax, redm[0]);
    atomic_max_pos(amax + 1, redm[1]);
  }
}

template <int DF>
__device__ __forceinline__ void store_grad4(void* dst_v, void* dst_lo_v, long off, float4 o,
                                            float gs_scale) {
  if constexpr (DF == PASE_FMT_F32) {
    st4(reinterpret_cast<float*>(dst_v) + off, o);
    if (dst_lo_v != nullptr)
      st4(reinterpret_cast<float*>(dst_lo_v) + off,
          make_float4(tf32_residual(o.x), tf32_residual(o.y), tf32_residual(o.z),
                      tf32_residual(o.w)));
  } else if constexpr (DF == PASE_FMT_BF16) {
    st4t(reinterpret_cast<__nv_bfloat16*>(dst_v) + off, o);
  } else {
    st4_f16x2(reinterpret_cast<__half*>(dst_v) + off, reinterpret_cast<__half*>(dst_lo_v) + off,
              make_float4(o.x * gs_scale, o.y * gs_scale, o.z * gs_scale, o.w * gs_scale));
  }
}

// pass 2 of pase_bn_prelu_bwd_apply_src for every utterance, into frames d_off/C + f of dst,
// f < d_span: the utterance's T frames, zeros in [T, d_span) and, for the first utterance,
// zeros in the `lead` frames before it.  Work item j < C/4 * ceil(T/RUN) computes a run; the
// others write the zero frames.  TRAIN: batch statistics over the pack, dy = gamma invstd (du -
// S1/count - xhat S2/count) with xhat = (y - mean) invstd; else eval mode (S1 = S2 = 0: dy =
// gamma invstd du; mean, S1, S2 unused).
template <typename YT, typename GT, int DF, bool TRAIN>
__device__ __forceinline__ void bn_prelu_bwd_apply_src_var_body(
    const YT* __restrict__ y, const int* __restrict__ tab, int C, const float* __restrict__ mean,
    const float* __restrict__ invstd, const float* __restrict__ gamma,
    const float* __restrict__ scale, const float* __restrict__ shift,
    const float* __restrict__ alpha, const double* __restrict__ S1,
    const double* __restrict__ S2, double inv_count, const void* A, long a_rs, int padL, int padR,
    const float* B, long b_rs, int b_shift, const float* pool, long p_rs, void* dst_v,
    void* dst_lo_v, int lead, double* __restrict__ dbias, const float* __restrict__ amax,
    float* __restrict__ scale_out) {
  pdl_wait();
  extern __shared__ double red[];
  float* redm = reinterpret_cast<float*>(red + C);
  for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.0;
  if (threadIdx.x == 0) redm[0] = 0.f;
  __syncthreads();
  float gs_scale = 1.f;
  if constexpr (DF == PASE_FMT_F16X2) {     // pase_bn_prelu_bwd_apply_src's bound
    const float mdu = amax[0];
    float b = 0.f;
    if constexpr (TRAIN) {
      const float mxh = amax[1];
      for (int i = threadIdx.x; i < C; i += blockDim.x) {
        const float gi = fabsf((gamma ? gamma[i] : 1.f) * invstd[i]);
        const float m1 = fabsf((float)(S1[i] * inv_count)), m2 = fabsf((float)(S2[i] * inv_count));
        b = fmaxf(b, gi * (mdu + m1 + mxh * m2));
      }
    } else {
      for (int i = threadIdx.x; i < C; i += blockDim.x)
        b = fmaxf(b, fabsf((gamma ? gamma[i] : 1.f) * invstd[i]) * mdu);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, off));
    if ((threadIdx.x & 31) == 0) atomic_max_pos(&redm[0], b);
    __syncthreads();
    gs_scale = f16_grad_scale(redm[0] * 1.0001f);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
      scale_out[0] = 1.f / gs_scale;
      scale_out[1] = gs_scale;
    }
  }
  const int* r = tab + BWD_ROW * blockIdx.y;
  const int T = __ldg(r);
  const long d_off = __ldg(r + 7);
  const int span = __ldg(r + 8), pre = blockIdx.y == 0 ? lead : 0;
  const int C4 = C >> 2;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c = (int)(idx % C4) * 4;
  const long run = idx / C4;
  const long nruns = (T + RUN - 1) / RUN;
  float acc[4] = {0, 0, 0, 0};
  if (run < nruns) {
    const BwdSrc s = var_src<GT>(r, A, a_rs, padL, padR, B, b_rs, b_shift, pool, p_rs);
    const YT* yn = y + __ldg(r + 1);
    const long t0 = run * RUN;
    const int nvalid = (T - (int)t0) < RUN ? (T - (int)t0) : RUN;
    float4 vs[RUN], gs[RUN];
#pragma unroll
    for (int i = 0; i < RUN; ++i) vs[i] = ld4t(yn + (long)((int)t0 + (i < nvalid ? i : 0)) * C + c);
    load_grad_run<GT>(s, 0, T, t0, nvalid, c, gs);
    float gi[4], scv[4], shv[4], alv[4], m1[4], m2[4], muv[4], isv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      gi[k] = (gamma ? gamma[c + k] : 1.f) * invstd[c + k];
      scv[k] = scale[c + k];
      shv[k] = shift[c + k];
      alv[k] = alpha[c + k];
      if constexpr (TRAIN) {
        m1[k] = (float)(S1[c + k] * inv_count);
        m2[k] = (float)(S2[c + k] * inv_count);
        muv[k] = mean[c + k];
        isv[k] = invstd[c + k];
      }
    }
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      if (i >= nvalid) break;
      const float vv[4] = {vs[i].x, vs[i].y, vs[i].z, vs[i].w};
      const float gg[4] = {gs[i].x, gs[i].y, gs[i].z, gs[i].w};
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float u = fmaf(vv[k], scv[k], shv[k]);
        const float du = u > 0.f ? gg[k] : alv[k] * gg[k];
        if constexpr (TRAIN) {
          const float xh = (vv[k] - muv[k]) * isv[k];
          o[k] = gi[k] * (du - m1[k] - xh * m2[k]);
        } else {
          o[k] = gi[k] * du;
        }
        acc[k] += o[k];
      }
      store_grad4<DF>(dst_v, dst_lo_v, d_off + ((long)t0 + i) * C + c,
                      make_float4(o[0], o[1], o[2], o[3]), gs_scale);
    }
    if (dbias) {
#pragma unroll
      for (int k = 0; k < 4; ++k) atomicAdd(&red[c + k], (double)acc[k]);
    }
  } else {
    // zero frames: [T, span), then [-pre, 0)
    const long z0 = (run - nruns) * RUN, tail = span - T;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < RUN; ++i) {
      const long j = z0 + i;
      const long f = j < tail ? T + j : j - tail - pre;
      if (j < tail + pre) store_grad4<DF>(dst_v, dst_lo_v, d_off + f * C + c, zero, gs_scale);
    }
  }
  if (dbias) {
    __syncthreads();
    if ((long)blockIdx.x * blockDim.x < (long)C4 * nruns)
      for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(dbias + i, red[i]);
  }
}

template <typename YT, typename GT, int DF>
__global__ void __launch_bounds__(THREADS)
bn_prelu_bwd_apply_src_var_kernel(const YT* __restrict__ y, const int* __restrict__ tab, int C,
                                  const float* __restrict__ invstd,
                                  const float* __restrict__ gamma,
                                  const float* __restrict__ scale, const float* __restrict__ shift,
                                  const float* __restrict__ alpha, const void* A, long a_rs,
                                  int padL, int padR, const float* B, long b_rs, int b_shift,
                                  const float* pool, long p_rs, void* dst_v, void* dst_lo_v,
                                  int lead, double* __restrict__ dbias,
                                  const float* __restrict__ amax, float* __restrict__ scale_out) {
  bn_prelu_bwd_apply_src_var_body<YT, GT, DF, false>(
      y, tab, C, nullptr, invstd, gamma, scale, shift, alpha, nullptr, nullptr, 0.0, A, a_rs,
      padL, padR, B, b_rs, b_shift, pool, p_rs, dst_v, dst_lo_v, lead, dbias, amax, scale_out);
}

template <typename YT, typename GT, int DF>
__global__ void __launch_bounds__(THREADS)
bn_prelu_bwd_apply_src_var_train_kernel(
    const YT* __restrict__ y, const int* __restrict__ tab, int C, const float* __restrict__ mean,
    const float* __restrict__ invstd, const float* __restrict__ gamma,
    const float* __restrict__ scale, const float* __restrict__ shift,
    const float* __restrict__ alpha, const double* __restrict__ S1,
    const double* __restrict__ S2, double inv_count, const void* A, long a_rs, int padL, int padR,
    const float* B, long b_rs, int b_shift, const float* pool, long p_rs, void* dst_v,
    void* dst_lo_v, int lead, double* __restrict__ dbias, const float* __restrict__ amax,
    float* __restrict__ scale_out) {
  bn_prelu_bwd_apply_src_var_body<YT, GT, DF, true>(
      y, tab, C, mean, invstd, gamma, scale, shift, alpha, S1, S2, inv_count, A, a_rs, padL, padR,
      B, b_rs, b_shift, pool, p_rs, dst_v, dst_lo_v, lead, dbias, amax, scale_out);
}

// g[row0 + t, c] = dout[o_off + c T + t] for tab rows {row0, T, o_off} (pase_out_bwd_reduce's
// layout change, one utterance per blockIdx.y)
__global__ void __launch_bounds__(256)
out_bwd_gather_var_kernel(const float* __restrict__ dout, const int* __restrict__ tab, int C,
                          float* __restrict__ g) {
  pdl_wait();
  const int* r = tab + 3 * blockIdx.y;
  const long row0 = __ldg(r), o = __ldg(r + 2);
  const int T = __ldg(r + 1);
  const long total = (long)T * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i / T), t = (int)(i - (long)c * T);
    g[(row0 + t) * C + c] = dout[o + i];
  }
}

// One window of a recording (WaveFe.encode_long): g[t*C + c] = dout[c*ld + col0 + t - c0] for
// the crop frames c0 <= t < c0+cn, 0 for the window's other frames t < T
__global__ void __launch_bounds__(256)
out_bwd_gather_crop_kernel(const float* __restrict__ dout, long ld, long col0, int T, int c0,
                           int cn, int C, float* __restrict__ g) {
  pdl_wait();
  const long total = (long)T * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i / T), t = (int)(i - (long)c * T);
    g[(long)t * C + c] = (t >= c0 && t < c0 + cn) ? dout[c * ld + col0 + (t - c0)] : 0.f;
  }
}

// ---- plain PReLU on (rows, C) ----
__global__ void prelu_fwd_kernel(const float* __restrict__ u, float* __restrict__ h,
                                 const float* __restrict__ alpha, long rows, int C, long ldu,
                                 long ldh) {
  const long total = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    h[r * ldh + c] = prelu1(u[r * ldu + c], alpha[c]);
  }
}

__global__ void __launch_bounds__(THREADS)
prelu_bwd_kernel(const float* __restrict__ u, const float* __restrict__ dh,
                 const float* __restrict__ alpha, float* __restrict__ du,
                 double* __restrict__ dalpha, long rows, int C, long ldu, long lddh, long lddu) {
  extern __shared__ double red[];     // [C] fp64 sums (order-independent to fp32 precision)
  for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.0;
  __syncthreads();
  // thread owns one channel of a strip of rows: coalesced over c
  const int cpb = min(C, (int)blockDim.x);         // channels covered per row pass
  const int rows_per_pass = blockDim.x / cpb;
  const int lc = threadIdx.x % cpb, lr = threadIdx.x / cpb;
  for (int c0 = 0; c0 < C; c0 += cpb) {
    const int c = c0 + lc;
    if (c >= C || lr >= rows_per_pass) continue;
    const float a = alpha[c];
    float acc = 0.f;
    for (long r = (long)blockIdx.x * rows_per_pass + lr; r < rows;
         r += (long)gridDim.x * rows_per_pass) {
      const float uu = u[r * ldu + c], g = dh[r * lddh + c];
      const bool pos = uu > 0.f;
      du[r * lddu + c] = pos ? g : a * g;
      acc += pos ? 0.f : uu * g;
    }
    atomicAdd(&red[c], (double)acc);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(dalpha + i, red[i]);
}


// out[c] (+)= sum_r X[r*ld + c]
__global__ void __launch_bounds__(THREADS)
colsum_kernel(const float* __restrict__ X, long ld, long rows, int C, double* __restrict__ acc) {
  pdl_wait();
  extern __shared__ double red[];     // [C] fp64 sums (order-independent to fp32 precision)
  for (int i = threadIdx.x; i < C; i += blockDim.x) red[i] = 0.0;
  __syncthreads();
  const int cpb = min(C, (int)blockDim.x);
  const int rows_per_pass = blockDim.x / cpb;
  const int lc = threadIdx.x % cpb, lr = threadIdx.x / cpb;
  for (int c0 = 0; c0 < C; c0 += cpb) {
    const int c = c0 + lc;
    if (c >= C || lr >= rows_per_pass) continue;
    // four independent partial sums: the loads of a thread's rows are in flight together
    const long step = (long)gridDim.x * rows_per_pass;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    long r = (long)blockIdx.x * rows_per_pass + lr;
    for (; r + 3 * step < rows; r += 4 * step) {
      a0 += X[r * ld + c];
      a1 += X[(r + step) * ld + c];
      a2 += X[(r + 2 * step) * ld + c];
      a3 += X[(r + 3 * step) * ld + c];
    }
    for (; r < rows; r += step) a0 += X[r * ld + c];
    atomicAdd(&red[c], (double)((a0 + a1) + (a2 + a3)));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(acc + i, red[i]);
}

__global__ void cast_d2f_kernel(const double* __restrict__ src, float* __restrict__ dst, int n,
                                float scale) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (float)(src[i] * (double)scale);
}

// ---- output affine + (N*T,C) -> (N,C,T) ----
// One 32 frames x 32 channels tile (blockIdx.x, blockIdx.y) of one utterance whose T frames are
// rows row0 .. row0+T-1 of y: h = y*scale+shift goes to o[c*ldo + t] and, when out_ntc is given,
// to the same rows of out_ntc.
__device__ __forceinline__ void out_affine_tile(const float* __restrict__ y,
                                                const float* __restrict__ scale,
                                                const float* __restrict__ shift,
                                                float* __restrict__ o, long ldo,
                                                float* __restrict__ out_ntc, long row0, int T,
                                                int C) {
  __shared__ float tile[32][33];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) {
      const float v = fmaf(y[(row0 + t) * C + c], scale[c], shift[c]);
      tile[i][threadIdx.x] = v;
      if (out_ntc) out_ntc[(row0 + t) * C + c] = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (t < T && c < C) o[(long)c * ldo + t] = tile[threadIdx.x][i];
  }
}

__global__ void out_affine_nct_kernel(const float* __restrict__ y, const float* __restrict__ scale,
                                      const float* __restrict__ shift, float* __restrict__ out,
                                      float* __restrict__ out_ntc, int T, int C) {
  pdl_wait();
  const int n = blockIdx.z;
  out_affine_tile(y, scale, shift, out + (long)n * C * T, T, out_ntc, (long)n * T, T, C);
}

// Packed variable-length output: blockIdx.y = utterance, tab row {y_row, T, out_off}; block
// (32, 8) owns 32 channels.  h = y*scale+shift as in out_affine_nct_kernel; the time mean of
// each channel is a double sum in a fixed order (8 strided partial sums, then added in order).
// mode 0: out (C,T) = h; 1: h - mean; 2: (2C,T) = [h ; mean]; 3: [h - mean ; mean].
__global__ void __launch_bounds__(256)
out_affine_var_kernel(const float* __restrict__ y, const float* __restrict__ scale,
                      const float* __restrict__ shift, float* __restrict__ out,
                      const int* __restrict__ tab, int C, int mode) {
  pdl_wait();
  __shared__ float tile[32][33];
  __shared__ double part[8][32];
  __shared__ float mean_s[32];
  const int* r = tab + 3 * blockIdx.y;
  const int T = __ldg(r + 1);
  const float* yn = y + (long)__ldg(r) * C;
  float* on = out + __ldg(r + 2);
  const int c0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  const int c = c0 + tx;
  const float sc = c < C ? scale[c] : 0.f, sh = c < C ? shift[c] : 0.f;
  if (mode != 0) {
    double s = 0.0;
    if (c < C)
      for (int t = ty; t < T; t += 8) s += (double)fmaf(yn[(long)t * C + c], sc, sh);
    part[ty][tx] = s;
    __syncthreads();
    if (ty == 0) {
      double m = 0.0;
      for (int k = 0; k < 8; ++k) m += part[k][tx];
      mean_s[tx] = (float)(m / (double)T);
    }
    __syncthreads();
  }
  const bool sub = mode == 1 || mode == 3, cat = mode >= 2;
  for (int t0 = 0; t0 < T; t0 += 32) {
    for (int i = ty; i < 32; i += 8) {
      const int t = t0 + i;
      if (t < T && c < C) {
        const float v = fmaf(yn[(long)t * C + c], sc, sh);
        tile[i][tx] = sub ? v - mean_s[tx] : v;
      }
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int cc = c0 + i, t = t0 + tx;
      if (t < T && cc < C) {
        on[(long)cc * T + t] = tile[tx][i];
        if (cat) on[(long)(C + cc) * T + t] = mean_s[i];
      }
    }
    __syncthreads();
  }
}

// Windowed output (StreamPool, so FeatureStream and WaveFe.extract_long): segment blockIdx.z's
// row {row0, T, ocol, ldo, col0} writes rows row0 .. row0+T-1 of y, as h = y*scale+shift, into
// columns col0 .. col0+T-1 of the (C, ldo) block that starts at element ocol*C of out.
__global__ void out_place_var_kernel(const float* __restrict__ y, const float* __restrict__ scale,
                                     const float* __restrict__ shift, float* __restrict__ out,
                                     const int* __restrict__ tab, int C) {
  pdl_wait();
  const int* row = tab + 5 * blockIdx.z;
  const int T = __ldg(row + 1);
  if ((int)blockIdx.x * 32 >= T) return;      // uniform over the block
  out_affine_tile(y, scale, shift, out + (long)__ldg(row + 2) * C + __ldg(row + 4), __ldg(row + 3),
                  nullptr, __ldg(row), T, C);
}

// select_output over a whole (C, T) output in place: one block per channel.  The time mean is
// a double sum in a fixed order (per-thread strided sums, then a fixed tree), so it does not
// depend on how the output was produced.  mode 1: h - mean; 2: rows C+c = mean; 3: both.
__global__ void __launch_bounds__(256)
out_select_kernel(float* __restrict__ out, long T, int C, int mode) {
  pdl_wait();
  __shared__ double part[256];
  __shared__ float mean_s;
  const int c = blockIdx.x, tid = threadIdx.x;
  float* row = out + (long)c * T;
  double s = 0.0;
  for (long t = tid; t < T; t += 256) s += (double)row[t];
  part[tid] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (tid < w) part[tid] += part[tid + w];
    __syncthreads();
  }
  if (tid == 0) mean_s = (float)(part[0] / (double)T);
  __syncthreads();
  const float m = mean_s;
  const bool sub = mode == 1 || mode == 3, cat = mode >= 2;
  float* mrow = out + (long)(C + c) * T;
  for (long t = tid; t < T; t += 256) {
    if (sub) row[t] -= m;
    if (cat) mrow[t] = m;
  }
}

// One 32 frames x 32 channels tile (blockIdx.x, blockIdx.y) of one utterance whose T frames are
// rows row0 .. row0+T-1 of g_ntc / y / dout_ntc and columns of the (C, T) block at dout + o:
// g = dout (0 when dout is null) + dout_ntc (when given), stored at g_ntc; S1 += g, S2 += g*xhat.
__device__ __forceinline__ void out_bwd_reduce_tile(const float* __restrict__ dout, long o,
                                                    const float* __restrict__ dout_ntc,
                                                    const float* __restrict__ y,
                                                    const float* __restrict__ mean,
                                                    const float* __restrict__ invstd, long row0,
                                                    int T, int C, float* __restrict__ g_ntc,
                                                    double* __restrict__ S1,
                                                    double* __restrict__ S2) {
  __shared__ float tile[32][33];
  __shared__ double r1[32], r2[32];   // fp64: order-independent to fp32 precision
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  if (threadIdx.y == 0) { r1[threadIdx.x] = 0.0; r2[threadIdx.x] = 0.0; }
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (dout && t < T && c < C) ? dout[o + (long)c * T + t] : 0.f;
  }
  __syncthreads();
  float a1 = 0.f, a2 = 0.f;
  const int c = c0 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i;
    if (t < T && c < C) {
      const long off = (row0 + t) * C + c;
      float g = tile[threadIdx.x][i];
      if (dout_ntc) g += dout_ntc[off];
      g_ntc[off] = g;
      const float xh = (y[off] - mean[c]) * invstd[c];
      a1 += g;
      a2 += g * xh;
    }
  }
  atomicAdd(&r1[threadIdx.x], (double)a1);
  atomicAdd(&r2[threadIdx.x], (double)a2);
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    atomicAdd(S1 + c, r1[threadIdx.x]);
    atomicAdd(S2 + c, r2[threadIdx.x]);
  }
}

// g[n,t,c] = dout_nct[n,c,t] (+ dout_ntc[n,t,c]); S1 += g, S2 += g*xhat
__global__ void out_bwd_reduce_kernel(const float* __restrict__ dout,
                                      const float* __restrict__ dout_ntc,
                                      const float* __restrict__ y, const float* __restrict__ mean,
                                      const float* __restrict__ invstd, int T, int C,
                                      float* __restrict__ g_ntc, double* __restrict__ S1,
                                      double* __restrict__ S2) {
  pdl_wait();
  const int n = blockIdx.z;
  out_bwd_reduce_tile(dout, (long)n * C * T, dout_ntc, y, mean, invstd, (long)n * T, T, C, g_ntc,
                      S1, S2);
}

// pase_out_bwd_reduce over packed utterances: tab rows {row0, T, o_off} (blockIdx.z), tiles of
// 32 frames x 32 channels; g_ntc[(row0 + t)*C + c] = dout[o_off + c*T + t], S1 += g,
// S2 += g*xhat
__global__ void out_bwd_reduce_var_kernel(const float* __restrict__ dout,
                                          const int* __restrict__ tab,
                                          const float* __restrict__ y,
                                          const float* __restrict__ mean,
                                          const float* __restrict__ invstd, int C,
                                          float* __restrict__ g_ntc, double* __restrict__ S1,
                                          double* __restrict__ S2) {
  pdl_wait();
  const int* r = tab + 3 * blockIdx.z;
  const int T = __ldg(r + 1);
  if ((int)blockIdx.x * 32 >= T) return;     // the whole block: before any barrier
  out_bwd_reduce_tile(dout, __ldg(r + 2), nullptr, y, mean, invstd, __ldg(r), T, C, g_ntc, S1, S2);
}

// in place on g (N*T,C): dy = scale_c*(g - use*(S1/M + xhat*S2/M))
__global__ void out_bwd_apply_kernel(float* __restrict__ g, const float* __restrict__ y,
                                     const float* __restrict__ mean,
                                     const float* __restrict__ invstd,
                                     const float* __restrict__ scale,
                                     const double* __restrict__ S1, const double* __restrict__ S2,
                                     double inv_count, int use_stats, long rows, int C) {
  pdl_wait();
  const long total = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float v = g[i];
    if (use_stats) {
      const float xh = (y[i] - mean[c]) * invstd[c];
      v = v - (float)(S1[c] * inv_count) - xh * (float)(S2[c] * inv_count);
    }
    g[i] = v * scale[c];
  }
}

__global__ void nct_to_ntc_kernel(const float* __restrict__ src, float* __restrict__ dst, int C,
                                  int T, long d_rs) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (t < T && c < C) tile[i][threadIdx.x] = src[((long)n * C + c) * T + t];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) dst[((long)n * T + t) * d_rs + c] = tile[threadIdx.x][i];
  }
}

__global__ void ntc_to_nct_kernel(const float* __restrict__ src, long s_rs,
                                  float* __restrict__ dst, int C, int T) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) tile[i][threadIdx.x] = src[((long)n * T + t) * s_rs + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (t < T && c < C) dst[((long)n * C + c) * T + t] = tile[threadIdx.x][i];
  }
}

__global__ void axpy_kernel(const float* __restrict__ x, float* __restrict__ y, long n, float a) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long)gridDim.x * blockDim.x)
    y[i] = fmaf(a, x[i], y[i]);
}

__global__ void scale_dev_kernel(float* __restrict__ x, long n, const float* __restrict__ s,
                                 float coef) {
  const float f = (s ? s[0] : 1.f) * coef;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long)gridDim.x * blockDim.x)
    x[i] *= f;
}

inline unsigned blocks_for(long total, int threads, int cap_mult = 8) {
  long b = (total + threads - 1) / threads;
  long cap = (long)pase_num_sms() * cap_mult;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// The operands of one BatchNorm/PReLU backward call (fields the entry point does not take
// stay zero / NULL).
BnStreamArgs bn_bwd_args(const void* y, int y_bf16, long y_ss, int N, int T, int C,
                         const void* srcA, int a_bf16, long a_ss, long a_rs, int padL, int padR,
                         const float* srcB, long b_ss, long b_rs, int b_shift, const float* pool,
                         long p_ss, long p_rs, int pool_d, int pool_T, void* dst, void* dst_lo,
                         int dst_fmt, long d_ss) {
  BnStreamArgs a{};
  a.y = y; a.y_bf16 = y_bf16; a.y_ss = y_ss; a.N = N; a.T = T; a.C = C;
  a.s = BwdSrc{srcA, a_ss, a_rs, padL, padR, srcB, b_ss, b_rs, b_shift,
               pool, p_ss, p_rs, pool ? pool_d : 0, pool_T};
  a.a_bf16 = a_bf16;
  a.dst = dst; a.dst_lo = dst_lo; a.dst_fmt = dst_fmt; a.d_ss = d_ss;
  return a;
}

// Which kernel runs a backward pass and how it is cut (also reported by pase_bn_bwd_plan).
//   pass 1 (pase_bn_prelu_bwd_reduce): staged when it writes only its sums (dst == NULL) and
//     pase_bn_stream_ok accepts the operands;
//   pass 2 (pase_bn_prelu_bwd_apply_src): staged when, in addition, dst / dst_lo take the
//     staged kernel's 16-byte stores; srcA == NULL: pase_bn_prelu_bwd_apply (stored du),
//     always the register kernel.
// Register kernels: one thread per run of `rows` time steps of a channel quad; when the
// grid stride keeps each thread on its channel quad, the grid is capped and threads loop.
struct BnBwdPlan {
  int path, rows;       // 0 register / 1 staged; time steps per work item
  long items, gx;       // work items (thread runs or tiles) of all samples; blocks per sample
  long blocks;          // blocks of the launch
};

BnBwdPlan bn_bwd_plan(const BnStreamArgs& a, int pass) {
  BnBwdPlan p{};
  bool staged = a.s.A != nullptr && pase_bn_stream_ok(a);
  if (pass == 1)
    staged = staged && a.dst == nullptr;
  else
    staged = staged && (a.d_ss % 8) == 0 && aligned16(a.dst) &&
             (a.dst_lo == nullptr || aligned16(a.dst_lo));
  if (staged) {
    const BnStreamPlan sp = pase_bn_stream_plan(a);
    p.path = 1; p.rows = sp.TT; p.items = sp.total; p.gx = sp.grid; p.blocks = sp.grid;
    return p;
  }
  const long threads = (long)(a.C / 4) * ((a.T + RUN - 1) / RUN);
  long gx = (threads + THREADS - 1) / THREADS;
  if ((THREADS % (a.C / 4)) == 0) {          // stride keeps the channel quad: cap the grid
    long cap = (8L * pase_num_sms() + a.N - 1) / a.N;
    if (cap < 1) cap = 1;
    if (gx > cap) gx = cap;
  }
  p.path = 0; p.rows = RUN; p.items = threads * a.N; p.gx = gx; p.blocks = gx * a.N;
  return p;
}

// The register kernels read and write every operand in quads of channels (a float4, or four
// 16-bit values in 8 bytes): pointers must be aligned to the quad's size and every row and
// sample stride must hold whole quads, else a kernel faults on a misaligned address.
#define PASE_CHECK_QUAD(fn, p, esz, name)                                                   \
  PASE_CHECK_ARG(((reinterpret_cast<uintptr_t>(p)) & (4u * (esz) - 1u)) == 0,                \
                 "%s: %s must be %d-byte aligned", fn, name, 4 * (int)(esz))
#define PASE_CHECK_STRIDE(fn, v, name)                                                      \
  PASE_CHECK_ARG(((v) % 4) == 0, "%s: %s=%ld must be a multiple of 4", fn, name, (long)(v))

// Checks of the operands of the three backward entry points, before any launch.  dst: du
// (pass 1, type of y) or dy (pass 2, format dst_fmt); du: the stored du of
// pase_bn_prelu_bwd_apply.
int bn_bwd_check(const char* fn, const BnStreamArgs& a, int pass, const void* du) {
  const int ysz = a.y_bf16 ? 2 : 4;
  PASE_CHECK_QUAD(fn, a.y, ysz, "y");
  PASE_CHECK_STRIDE(fn, a.y_ss, "y_sample_stride");
  if (a.s.A) {
    PASE_CHECK_QUAD(fn, a.s.A, a.a_bf16 ? 2 : 4, "srcA");
    PASE_CHECK_STRIDE(fn, a.s.a_ss, "a_sample_stride");
    PASE_CHECK_STRIDE(fn, a.s.a_rs, "a_row_stride");
    PASE_CHECK_ARG(a.s.a_rs >= a.C, "%s: a_row_stride=%ld < C=%d", fn, a.s.a_rs, a.C);
  }
  if (a.s.B) {
    PASE_CHECK_QUAD(fn, a.s.B, 4, "srcB");
    PASE_CHECK_STRIDE(fn, a.s.b_ss, "b_sample_stride");
    PASE_CHECK_STRIDE(fn, a.s.b_rs, "b_row_stride");
    PASE_CHECK_ARG(a.s.b_rs >= a.C, "%s: b_row_stride=%ld < C=%d", fn, a.s.b_rs, a.C);
  }
  if (a.s.P && a.s.pool_d != 0) {
    PASE_CHECK_QUAD(fn, a.s.P, 4, "pool");
    PASE_CHECK_STRIDE(fn, a.s.p_ss, "pool_sample_stride");
    PASE_CHECK_STRIDE(fn, a.s.p_rs, "pool_row_stride");
    PASE_CHECK_ARG(a.s.pool_d > 0 && a.s.pool_T >= 0 && (long)a.s.pool_T * a.s.pool_d <= a.T,
                   "%s: pool_T=%d x pool_d=%d exceeds T=%d", fn, a.s.pool_T, a.s.pool_d, a.T);
  }
  const int dsz = pass == 1 ? ysz : (a.dst_fmt == PASE_FMT_F32 ? 4 : 2);
  if (a.dst) {
    PASE_CHECK_QUAD(fn, a.dst, dsz, "dst");
    PASE_CHECK_STRIDE(fn, a.d_ss, "dst_sample_stride");
  }
  if (a.dst_lo) PASE_CHECK_QUAD(fn, a.dst_lo, dsz, "dst_lo");
  if (du) PASE_CHECK_QUAD(fn, du, ysz, "du");
  return PASE_OK;
}

}  // namespace

extern "C" {

int pase_reflect_pad_wave(const float* x, void* dst, void* dst_lo, int dst_fmt, int N, int T,
                          int padL, int padR, long pitch, void* stream) {
  PASE_CHECK_ARG(x && dst && N > 0 && T > 0, "pase_reflect_pad_wave: bad args");
  PASE_CHECK_ARG(padL < T && padR < T, "pase_reflect_pad_wave: reflect pad (%d,%d) >= T=%d", padL,
                 padR, T);
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2 && (dst_fmt != PASE_FMT_F16X2 || dst_lo),
                 "pase_reflect_pad_wave: bad dst_fmt %d / missing lo", dst_fmt);
  const int Tp = T + padL + padR;
  PASE_CHECK_ARG(pitch >= Tp, "pase_reflect_pad_wave: pitch %ld < padded length %d", pitch, Tp);
  dim3 grid(blocks_for(Tp, 256, 4), N);
  with_fmt(dst_fmt, [&](auto df) {
    PASE_LAUNCH((reflect_pad_wave_kernel<decltype(df)::value>), grid, 256, 0, stream, x, dst,
                dst_lo, T, padL, Tp, pitch);
  });
  PASE_LAUNCH_CHECK("pase_reflect_pad_wave");
  return PASE_OK;
}

int pase_reflect_pad_wave_var(const float* x, const int* tab, int nseg, int max_T, void* dst,
                              void* dst_lo, int dst_fmt, int padL, int padR, void* stream) {
  PASE_CHECK_ARG(x && tab && dst && nseg > 0 && nseg <= 65535 && max_T > 0,
                 "pase_reflect_pad_wave_var: bad args (nseg=%d max_T=%d)", nseg, max_T);
  PASE_CHECK_ARG(padL < max_T && padR < max_T && padL >= 0 && padR >= 0,
                 "pase_reflect_pad_wave_var: reflect pad (%d,%d)", padL, padR);
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2 && (dst_fmt != PASE_FMT_F16X2 || dst_lo),
                 "pase_reflect_pad_wave_var: bad dst_fmt %d / missing lo", dst_fmt);
  dim3 grid(blocks_for((long)max_T + padL + padR, 256, 4), nseg);
  with_fmt(dst_fmt, [&](auto df) {
    PASE_LAUNCH((reflect_pad_wave_var_kernel<decltype(df)::value>), grid, 256, 0, stream, x, tab,
                dst, dst_lo, padL, padR);
  });
  PASE_LAUNCH_CHECK("pase_reflect_pad_wave_var");
  return PASE_OK;
}

int pase_bn_finalize(const double* colsum, const double* colsumsq, int C, int fold, double count,
                     const float* gamma, const float* beta, float* running_mean,
                     float* running_var, float momentum, float eps, float* mean, float* invstd,
                     float* scale, float* shift, void* stream) {
  PASE_CHECK_ARG(colsum && colsumsq && mean && invstd && scale && shift && C > 0 && fold > 0,
                 "pase_bn_finalize: bad args");
  PASE_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr),
                 "pase_bn_finalize: running stats must be given together");
  PASE_LAUNCH((bn_finalize_kernel), (C + 127) / 128, 128, 0, (cudaStream_t)stream, 
      colsum, colsumsq, C, fold, count, gamma, beta, running_mean, running_var, momentum, eps,
      mean, invstd, scale, shift);
  PASE_LAUNCH_CHECK("pase_bn_finalize");
  return PASE_OK;
}

int pase_bn_eval_affine(const float* running_mean, const float* running_var, const float* gamma,
                        const float* beta, int C, float eps, float* mean, float* invstd,
                        float* scale, float* shift, void* stream) {
  PASE_CHECK_ARG(running_mean && running_var && C > 0, "pase_bn_eval_affine: bad args");
  bn_eval_affine_kernel<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      running_mean, running_var, gamma, beta, C, eps, mean, invstd, scale, shift);
  PASE_LAUNCH_CHECK("pase_bn_eval_affine");
  return PASE_OK;
}

int pase_bn_prelu_pad_fwd(const void* y, int y_bf16, long y_sample_stride, int N, int T, int C,
                          const float* scale, const float* shift, const float* alpha, void* dst,
                          void* dst_lo, int dst_fmt, long dst_sample_stride, long dst_row_stride,
                          int padL, int padR, float* pool, long pool_sample_stride,
                          long pool_row_stride, int pool_d, int pool_T, void* stream) {
  PASE_CHECK_ARG(y && dst && scale && shift && alpha, "pase_bn_prelu_pad_fwd: null pointer");
  PASE_CHECK_ARG(N > 0 && T > 0 && C > 0 && (C % 4) == 0,
                 "pase_bn_prelu_pad_fwd: C=%d must be a positive multiple of 4", C);
  PASE_CHECK_ARG((padL == 0 && padR == 0) || (padL < T && padR < T),
                 "pase_bn_prelu_pad_fwd: reflect pad (%d,%d) >= T=%d", padL, padR, T);
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2 && (dst_fmt != PASE_FMT_F16X2 || dst_lo),
                 "pase_bn_prelu_pad_fwd: bad dst_fmt %d / missing lo", dst_fmt);
  {
    const char* fn = "pase_bn_prelu_pad_fwd";
    const int dsz = dst_fmt == PASE_FMT_F32 ? 4 : 2;
    PASE_CHECK_QUAD(fn, y, y_bf16 ? 2 : 4, "y");
    PASE_CHECK_STRIDE(fn, y_sample_stride, "y_sample_stride");
    PASE_CHECK_QUAD(fn, dst, dsz, "dst");
    if (dst_lo) PASE_CHECK_QUAD(fn, dst_lo, dsz, "dst_lo");
    PASE_CHECK_STRIDE(fn, dst_sample_stride, "dst_sample_stride");
    PASE_CHECK_STRIDE(fn, dst_row_stride, "dst_row_stride");
    if (pool && pool_d != 0) {
      PASE_CHECK_QUAD(fn, pool, 4, "pool");
      PASE_CHECK_STRIDE(fn, pool_sample_stride, "pool_sample_stride");
      PASE_CHECK_STRIDE(fn, pool_row_stride, "pool_row_stride");
      PASE_CHECK_ARG(pool_d > 0 && pool_T >= 0 && (long)pool_T * pool_d <= T,
                     "%s: pool_T=%d x pool_d=%d exceeds T=%d", fn, pool_T, pool_d, T);
    }
  }
  if (pool == nullptr) pool_d = 0;
  const int Tp = T + padL + padR;
  const long threads = (long)(C / 4) * fwd_runs(Tp, padL, pool_d, pool_T).total;
  dim3 grid((unsigned)((threads + FWD_THREADS - 1) / FWD_THREADS), N);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_FWD(YT, DF)                                                                       \
  PASE_LAUNCH((bn_prelu_pad_fwd_kernel<YT, DF>), grid, FWD_THREADS, 0, st,                     \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, scale, shift, alpha, dst,         \
      dst_sample_stride, dst_row_stride, padL, Tp, pool, pool_sample_stride, pool_row_stride,  \
      pool_d, pool_T, dst_lo)
  if (y_bf16) {
    if (dst_fmt == PASE_FMT_F32) PASE_FWD(__nv_bfloat16, PASE_FMT_F32);
    else if (dst_fmt == PASE_FMT_BF16) PASE_FWD(__nv_bfloat16, PASE_FMT_BF16);
    else PASE_FWD(__nv_bfloat16, PASE_FMT_F16X2);
  } else {
    if (dst_fmt == PASE_FMT_F32) PASE_FWD(float, PASE_FMT_F32);
    else if (dst_fmt == PASE_FMT_BF16) PASE_FWD(float, PASE_FMT_BF16);
    else PASE_FWD(float, PASE_FMT_F16X2);
  }
#undef PASE_FWD
  PASE_LAUNCH_CHECK("pase_bn_prelu_pad_fwd");
  return PASE_OK;
}

int pase_bn_prelu_pad_fwd_var(const void* y, int y_bf16, const int* tab, int nseg, int max_T,
                              int C, const float* scale, const float* shift, const float* alpha,
                              void* dst, void* dst_lo, int dst_fmt, long dst_row_stride,
                              int padL, int padR, float* pool, long pool_row_stride, int sep,
                              void* stream) {
  const char* fn = "pase_bn_prelu_pad_fwd_var";
  PASE_CHECK_ARG(y && tab && dst && scale && shift && alpha, "%s: null pointer", fn);
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && max_T > 0 && C > 0 && (C % 4) == 0,
                 "%s: nseg=%d max_T=%d C=%d (C a positive multiple of 4)", fn, nseg, max_T, C);
  PASE_CHECK_ARG(padL >= 0 && padR >= 0, "%s: reflect pad (%d,%d)", fn, padL, padR);
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2 && (dst_fmt != PASE_FMT_F16X2 || dst_lo),
                 "%s: bad dst_fmt %d / missing lo", fn, dst_fmt);
  {
    const int dsz = dst_fmt == PASE_FMT_F32 ? 4 : 2;
    PASE_CHECK_QUAD(fn, y, y_bf16 ? 2 : 4, "y");
    PASE_CHECK_QUAD(fn, dst, dsz, "dst");
    if (dst_lo) PASE_CHECK_QUAD(fn, dst_lo, dsz, "dst_lo");
    PASE_CHECK_STRIDE(fn, dst_row_stride, "dst_row_stride");
    if (pool) {
      PASE_CHECK_QUAD(fn, pool, 4, "pool");
      PASE_CHECK_STRIDE(fn, pool_row_stride, "pool_row_stride");
    }
  }
  // each utterance's pool_d / pool_T live in the device table: size for the most runs any
  // T <= max_T can need (cutting [0, Tp) into three ranges adds at most two partial runs, and
  // a pooled run is never shorter than RUN)
  const long threads = (long)(C / 4) * (((long)max_T + padL + padR + RUN - 1) / RUN + 2);
  dim3 grid((unsigned)((threads + FWD_THREADS - 1) / FWD_THREADS), nseg);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_FWD(YT, DF)                                                                       \
  PASE_LAUNCH((bn_prelu_pad_fwd_var_kernel<YT, DF>), grid, FWD_THREADS, 0, st,                 \
      reinterpret_cast<const YT*>(y), tab, C, scale, shift, alpha, dst, dst_row_stride, padL,  \
      padR, pool, pool_row_stride, sep, dst_lo)
  if (y_bf16) {
    if (dst_fmt == PASE_FMT_F32) PASE_FWD(__nv_bfloat16, PASE_FMT_F32);
    else if (dst_fmt == PASE_FMT_BF16) PASE_FWD(__nv_bfloat16, PASE_FMT_BF16);
    else PASE_FWD(__nv_bfloat16, PASE_FMT_F16X2);
  } else {
    if (dst_fmt == PASE_FMT_F32) PASE_FWD(float, PASE_FMT_F32);
    else if (dst_fmt == PASE_FMT_BF16) PASE_FWD(float, PASE_FMT_BF16);
    else PASE_FWD(float, PASE_FMT_F16X2);
  }
#undef PASE_FWD
  PASE_LAUNCH_CHECK(fn);
  return PASE_OK;
}

int pase_bn_prelu_bwd_reduce(const void* y, int y_bf16, long y_sample_stride, int N, int T, int C,
                             const float* mean, const float* invstd, const float* scale,
                             const float* shift, const float* alpha, const void* srcA,
                             int a_bf16, long a_sample_stride, long a_row_stride, int padL,
                             int padR, const float* srcB, long b_sample_stride,
                             long b_row_stride, int b_shift, const float* pool,
                             long pool_sample_stride, long pool_row_stride, int pool_d,
                             int pool_T, void* dst, long dst_sample_stride, double* S1,
                             double* S2, double* dalpha, float* amax, void* stream) {
  PASE_CHECK_ARG(y && mean && invstd && scale && shift && alpha && S1 && S2 && dalpha && srcA,
                 "pase_bn_prelu_bwd_reduce: null pointer (srcA is mandatory; dst may be NULL: "
                 "sums only, see pase_bn_prelu_bwd_apply_src)");
  PASE_CHECK_ARG(N > 0 && T > 0 && C > 0 && (C % 4) == 0 && C <= 4096,
                 "pase_bn_prelu_bwd_reduce: C=%d must be a multiple of 4, <= 4096", C);
  BnStreamArgs sa = bn_bwd_args(y, y_bf16, y_sample_stride, N, T, C, srcA, a_bf16,
                                a_sample_stride, a_row_stride, padL, padR, srcB, b_sample_stride,
                                b_row_stride, b_shift, pool, pool_sample_stride, pool_row_stride,
                                pool_d, pool_T, dst, nullptr, 0, dst_sample_stride);
  const int rc = bn_bwd_check("pase_bn_prelu_bwd_reduce", sa, 1, nullptr);
  if (rc != PASE_OK) return rc;
  const BwdSrc& s = sa.s;
  const BnBwdPlan plan = bn_bwd_plan(sa, 1);
  if (plan.path == 1) {                    // sums only: persistent staged kernel
    sa.mean = mean; sa.invstd = invstd; sa.scale = scale; sa.shift = shift; sa.alpha = alpha;
    sa.S1 = S1; sa.S2 = S2; sa.dalpha = dalpha; sa.amax = amax;
    return pase_bn_stream_reduce(sa, (cudaStream_t)stream);
  }
  dim3 grid((unsigned)plan.gx, N);
  const size_t sm = 3 * C * sizeof(double) + 2 * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  // C >= 2048: the block sums need more than the default 48 KB of dynamic shared memory
#define PASE_RED(YT, GT)                                                                     \
  do {                                                                                       \
    if (sm > 48 * 1024)                                                                      \
      cudaFuncSetAttribute(bn_prelu_bwd_reduce_kernel<YT, GT>,                               \
                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);            \
    bn_prelu_bwd_reduce_kernel<YT, GT><<<grid, THREADS, sm, st>>>(                           \
        reinterpret_cast<const YT*>(y), y_sample_stride, T, C, mean, invstd, scale, shift,   \
        alpha, s, reinterpret_cast<YT*>(dst), dst_sample_stride, S1, S2, dalpha, amax);      \
  } while (0)
  if (y_bf16) {
    if (a_bf16) PASE_RED(__nv_bfloat16, __nv_bfloat16);
    else PASE_RED(__nv_bfloat16, float);
  } else {
    if (a_bf16) PASE_RED(float, __nv_bfloat16);
    else PASE_RED(float, float);
  }
#undef PASE_RED
  PASE_LAUNCH_CHECK("pase_bn_prelu_bwd_reduce");
  return PASE_OK;
}

int pase_bn_prelu_bwd_apply(const void* y, int y_bf16, long y_sample_stride, int N, int T, int C,
                            const float* mean, const float* invstd, const float* gamma,
                            const double* S1, const double* S2, double count, const void* du,
                            void* dst, void* dst_lo, int dst_fmt, long dst_sample_stride,
                            double* dbias_acc, const float* amax, float* scale_out,
                            void* stream) {
  PASE_CHECK_ARG(y && mean && invstd && S1 && S2 && du && dst,
                 "pase_bn_prelu_bwd_apply: null pointer");
  PASE_CHECK_ARG(N > 0 && T > 0 && C > 0 && (C % 4) == 0 && C <= 4096,
                 "pase_bn_prelu_bwd_apply: bad C=%d", C);
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2, "pase_bn_prelu_bwd_apply: bad dst_fmt %d", dst_fmt);
  PASE_CHECK_ARG(dst_fmt != PASE_FMT_F16X2 || (dst_lo && amax && scale_out && !y_bf16),
                 "pase_bn_prelu_bwd_apply: the fp16-pair format needs dst_lo, amax, scale_out "
                 "and fp32 y/du");
  PASE_CHECK_ARG((dst_fmt == PASE_FMT_BF16) == (y_bf16 != 0),
                 "pase_bn_prelu_bwd_apply: bf16 y/du goes with bf16 dst (and only with it)");
  const BnStreamArgs sa = bn_bwd_args(y, y_bf16, y_sample_stride, N, T, C, nullptr, 0, 0, 0, 0,
                                      0, nullptr, 0, 0, 0, nullptr, 0, 0, 0, 0, dst, dst_lo,
                                      dst_fmt, dst_sample_stride);
  const int rc = bn_bwd_check("pase_bn_prelu_bwd_apply", sa, 2, du);
  if (rc != PASE_OK) return rc;
  const BnBwdPlan plan = bn_bwd_plan(sa, 2);          // always the register kernel
  dim3 grid((unsigned)plan.gx, N);
  const size_t sm = C * sizeof(double) + sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_APP(YT, DF)                                                                      \
  bn_prelu_bwd_apply_kernel<YT, DF><<<grid, THREADS, sm, st>>>(                               \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, mean, invstd, gamma, S1, S2,     \
      1.0 / count, reinterpret_cast<const YT*>(du), dst, dst_sample_stride, dbias_acc,        \
      dst_lo, amax, scale_out)
  if (dst_fmt == PASE_FMT_BF16) PASE_APP(__nv_bfloat16, PASE_FMT_BF16);
  else if (dst_fmt == PASE_FMT_F16X2) PASE_APP(float, PASE_FMT_F16X2);
  else PASE_APP(float, PASE_FMT_F32);
#undef PASE_APP
  PASE_LAUNCH_CHECK("pase_bn_prelu_bwd_apply");
  return PASE_OK;
}

int pase_bn_prelu_bwd_apply_src(const void* y, int y_bf16, long y_sample_stride, int N, int T,
                                int C, const float* mean, const float* invstd,
                                const float* gamma, const float* scale, const float* shift,
                                const float* alpha, const double* S1, const double* S2,
                                double count, const void* srcA, int a_bf16, long a_sample_stride,
                                long a_row_stride, int padL, int padR, const float* srcB,
                                long b_sample_stride, long b_row_stride, int b_shift,
                                const float* pool, long pool_sample_stride, long pool_row_stride,
                                int pool_d, int pool_T, void* dst, void* dst_lo, int dst_fmt,
                                long dst_sample_stride, double* dbias_acc, const float* amax,
                                float* scale_out, void* stream) {
  PASE_CHECK_ARG(y && mean && invstd && scale && shift && alpha && S1 && S2 && srcA && dst,
                 "pase_bn_prelu_bwd_apply_src: null pointer");
  PASE_CHECK_ARG(N > 0 && T > 0 && C > 0 && (C % 4) == 0 && C <= 4096,
                 "pase_bn_prelu_bwd_apply_src: bad C=%d", C);
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2, "pase_bn_prelu_bwd_apply_src: bad dst_fmt %d",
                 dst_fmt);
  PASE_CHECK_ARG(dst_fmt != PASE_FMT_F16X2 || (dst_lo && amax && scale_out && !y_bf16),
                 "pase_bn_prelu_bwd_apply_src: the fp16-pair format needs dst_lo, amax, "
                 "scale_out and fp32 y");
  PASE_CHECK_ARG((dst_fmt == PASE_FMT_BF16) == (y_bf16 != 0),
                 "pase_bn_prelu_bwd_apply_src: bf16 y goes with bf16 dst (and only with it)");
  PASE_CHECK_ARG(!a_bf16 || y_bf16, "pase_bn_prelu_bwd_apply_src: bf16 srcA needs bf16 y");
  BnStreamArgs sa = bn_bwd_args(y, y_bf16, y_sample_stride, N, T, C, srcA, a_bf16,
                                a_sample_stride, a_row_stride, padL, padR, srcB, b_sample_stride,
                                b_row_stride, b_shift, pool, pool_sample_stride, pool_row_stride,
                                pool_d, pool_T, dst, dst_lo, dst_fmt, dst_sample_stride);
  const int rc = bn_bwd_check("pase_bn_prelu_bwd_apply_src", sa, 2, nullptr);
  if (rc != PASE_OK) return rc;
  const BwdSrc& s = sa.s;
  const BnBwdPlan plan = bn_bwd_plan(sa, 2);
  if (plan.path == 1) {
    sa.mean = mean; sa.invstd = invstd; sa.gamma = gamma; sa.scale = scale; sa.shift = shift;
    sa.alpha = alpha; sa.S1in = S1; sa.S2in = S2; sa.inv_count = 1.0 / count;
    sa.dbias = dbias_acc; sa.amax = const_cast<float*>(amax); sa.scale_out = scale_out;
    return pase_bn_stream_apply(sa, (cudaStream_t)stream);
  }
  dim3 grid((unsigned)plan.gx, N);
  const size_t sm = C * sizeof(double) + sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_APS(YT, GT, DF)                                                                   \
  bn_prelu_bwd_apply_src_kernel<YT, GT, DF><<<grid, THREADS, sm, st>>>(                        \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, mean, invstd, gamma, scale, shift, \
      alpha, S1, S2, 1.0 / count, s, dst, dst_sample_stride, dbias_acc, dst_lo, amax, scale_out)
  if (dst_fmt == PASE_FMT_BF16) {
    if (a_bf16) PASE_APS(__nv_bfloat16, __nv_bfloat16, PASE_FMT_BF16);
    else PASE_APS(__nv_bfloat16, float, PASE_FMT_BF16);
  } else if (dst_fmt == PASE_FMT_F16X2) {
    PASE_APS(float, float, PASE_FMT_F16X2);
  } else {
    PASE_APS(float, float, PASE_FMT_F32);
  }
#undef PASE_APS
  PASE_LAUNCH_CHECK("pase_bn_prelu_bwd_apply_src");
  return PASE_OK;
}

int pase_bn_bwd_plan(int pass, const void* y, int y_bf16, long y_sample_stride, int N, int T,
                     int C, const void* srcA, int a_bf16, long a_sample_stride,
                     long a_row_stride, int padL, int padR, const float* srcB,
                     long b_sample_stride, long b_row_stride, int b_shift, const float* pool,
                     long pool_sample_stride, long pool_row_stride, int pool_d, int pool_T,
                     void* dst, void* dst_lo, int dst_fmt, long dst_sample_stride, long* out4) {
  PASE_CHECK_ARG(out4 && y && (pass == 1 || pass == 2) && (pass == 2 || srcA),
                 "pase_bn_bwd_plan: bad args");
  PASE_CHECK_ARG(N > 0 && T > 0 && C > 0 && (C % 4) == 0 && C <= 4096,
                 "pase_bn_bwd_plan: C=%d must be a multiple of 4, <= 4096", C);
  PASE_CHECK_ARG(pass == 1 || (dst && dst_fmt >= 0 && dst_fmt <= 2),
                 "pase_bn_bwd_plan: pass 2 needs dst and a dst_fmt in 0..2");
  const BnStreamArgs sa = bn_bwd_args(y, y_bf16, y_sample_stride, N, T, C, srcA, a_bf16,
                                      a_sample_stride, a_row_stride, padL, padR, srcB,
                                      b_sample_stride, b_row_stride, b_shift, pool,
                                      pool_sample_stride, pool_row_stride, pool_d, pool_T, dst,
                                      pass == 1 ? nullptr : dst_lo, dst_fmt, dst_sample_stride);
  const int rc = bn_bwd_check("pase_bn_bwd_plan", sa, pass, nullptr);
  if (rc != PASE_OK) return rc;
  const BnBwdPlan p = bn_bwd_plan(sa, pass);
  out4[0] = p.path;
  out4[1] = p.rows;
  out4[2] = p.items;
  out4[3] = p.blocks;
  return PASE_OK;
}

int pase_prelu_fwd(const float* u, float* h, const float* alpha, long rows, int C, long ldu,
                   long ldh, void* stream) {
  PASE_CHECK_ARG(u && h && alpha && rows > 0 && C > 0, "pase_prelu_fwd: bad args");
  prelu_fwd_kernel<<<blocks_for(rows * C, 256), 256, 0, (cudaStream_t)stream>>>(u, h, alpha, rows,
                                                                                C, ldu, ldh);
  PASE_LAUNCH_CHECK("pase_prelu_fwd");
  return PASE_OK;
}

int pase_prelu_bwd(const float* u, const float* dh, const float* alpha, float* du, double* dalpha,
                   long rows, int C, long ldu, long lddh, long lddu, void* stream) {
  PASE_CHECK_ARG(u && dh && alpha && du && dalpha && rows > 0 && C > 0 && C <= 6144,
                 "pase_prelu_bwd: bad args");
  const int cpb = C < THREADS ? C : THREADS;
  const int rpp = THREADS / cpb;
  long nb = (rows + rpp - 1) / rpp;
  long cap = (long)pase_num_sms() * 4;
  if (nb > cap) nb = cap;
  prelu_bwd_kernel<<<(unsigned)nb, THREADS, C * sizeof(double), (cudaStream_t)stream>>>(
      u, dh, alpha, du, dalpha, rows, C, ldu, lddh, lddu);
  PASE_LAUNCH_CHECK("pase_prelu_bwd");
  return PASE_OK;
}

int pase_colsum(const float* X, long ld, long rows, int C, double* acc, void* stream) {
  PASE_CHECK_ARG(X && acc && rows > 0 && C > 0, "pase_colsum: bad args");
  // wide matrices (e.g. the 21525-column lps head) are processed in column panels
  for (int c0 = 0; c0 < C; c0 += 4096) {
    const int Cp = (C - c0) < 4096 ? (C - c0) : 4096;
    const int cpb = Cp < THREADS ? Cp : THREADS;
    const int rpp = THREADS / cpb;
    long nb = (rows + rpp * 8 - 1) / (rpp * 8);
    // every block ends with C same-address fp64 atomics per column: one block per SM keeps
    // that tail short for small matrices (12.2 -> 6.5 us at 6 MB); large ones need the
    // blocks for streaming (39 MB: 19.9 us at 4 per SM, 37 us at 1 per SM)
    long per_sm = rows * (long)Cp * 4 / (8L << 20);
    per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
    long cap = (long)pase_num_sms() * per_sm;
    if (nb > cap) nb = cap;
    if (nb < 1) nb = 1;
    PASE_LAUNCH((colsum_kernel), (unsigned)nb, THREADS, Cp * sizeof(double), (cudaStream_t)stream, 
        X + c0, ld, rows, Cp, acc + c0);
    PASE_LAUNCH_CHECK("pase_colsum");
  }
  return PASE_OK;
}

int pase_cast_d2f(const double* src, float* dst, int n, float scale, void* stream) {
  PASE_CHECK_ARG(src && dst && n > 0, "pase_cast_d2f: bad args");
  PASE_LAUNCH((cast_d2f_kernel), (n + 255) / 256, 256, 0, (cudaStream_t)stream, src, dst, n, scale);
  PASE_LAUNCH_CHECK("pase_cast_d2f");
  return PASE_OK;
}

int pase_out_affine_nct(const float* y, const float* scale, const float* shift, float* out,
                        float* out_ntc, int N, int T, int C, void* stream) {
  PASE_CHECK_ARG(y && scale && shift && out && N > 0 && T > 0 && C > 0,
                 "pase_out_affine_nct: bad args");
  dim3 grid((T + 31) / 32, (C + 31) / 32, N), block(32, 8);
  PASE_LAUNCH((out_affine_nct_kernel), grid, block, 0, (cudaStream_t)stream, y, scale, shift, out, out_ntc, T,
                                                                  C);
  PASE_LAUNCH_CHECK("pase_out_affine_nct");
  return PASE_OK;
}

int pase_out_affine_var(const float* y, const float* scale, const float* shift, float* out,
                        const int* tab, int nseg, int C, int mode, void* stream) {
  PASE_CHECK_ARG(y && scale && shift && out && tab && C > 0, "pase_out_affine_var: bad args");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535, "pase_out_affine_var: nseg=%d", nseg);
  PASE_CHECK_ARG(mode >= 0 && mode <= 3, "pase_out_affine_var: mode %d", mode);
  PASE_LAUNCH((out_affine_var_kernel), dim3((C + 31) / 32, nseg), dim3(32, 8), 0,
              (cudaStream_t)stream, y, scale, shift, out, tab, C, mode);
  PASE_LAUNCH_CHECK("pase_out_affine_var");
  return PASE_OK;
}

int pase_out_place_var(const float* y, const float* scale, const float* shift, float* out,
                       const int* tab, int nseg, int max_T, int C, void* stream) {
  PASE_CHECK_ARG(y && scale && shift && out && tab && max_T > 0 && C > 0,
                 "pase_out_place_var: bad args");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535, "pase_out_place_var: nseg=%d", nseg);
  PASE_LAUNCH((out_place_var_kernel), dim3((max_T + 31) / 32, (C + 31) / 32, nseg), dim3(32, 8),
              0, (cudaStream_t)stream, y, scale, shift, out, tab, C);
  PASE_LAUNCH_CHECK("pase_out_place_var");
  return PASE_OK;
}

int pase_out_select(float* out, long T, int C, int mode, void* stream) {
  PASE_CHECK_ARG(out && T > 0 && C > 0, "pase_out_select: bad args");
  PASE_CHECK_ARG(mode >= 1 && mode <= 3, "pase_out_select: mode %d", mode);
  PASE_LAUNCH((out_select_kernel), dim3(C), 256, 0, (cudaStream_t)stream, out, T, C, mode);
  PASE_LAUNCH_CHECK("pase_out_select");
  return PASE_OK;
}

int pase_out_bwd_reduce(const float* dout, const float* dout_ntc, const float* y,
                        const float* mean, const float* invstd, int N, int T, int C, float* g_ntc,
                        double* S1, double* S2, void* stream) {
  PASE_CHECK_ARG((dout || dout_ntc) && y && mean && invstd && g_ntc && S1 && S2,
                 "pase_out_bwd_reduce: null pointer");
  PASE_CHECK_ARG(N > 0 && T > 0 && C > 0, "pase_out_bwd_reduce: N=%d T=%d C=%d", N, T, C);
  dim3 grid((T + 31) / 32, (C + 31) / 32, N), block(32, 8);
  PASE_LAUNCH((out_bwd_reduce_kernel), grid, block, 0, (cudaStream_t)stream, dout, dout_ntc, y, mean, invstd,
                                                                  T, C, g_ntc, S1, S2);
  PASE_LAUNCH_CHECK("pase_out_bwd_reduce");
  return PASE_OK;
}

int pase_out_bwd_apply(float* g, const float* y, const float* mean, const float* invstd,
                       const float* scale, const double* S1, const double* S2, double count,
                       int use_stats, long rows, int C, void* stream) {
  PASE_CHECK_ARG(g && y && mean && invstd && scale && S1 && S2 && rows > 0 && C > 0,
                 "pase_out_bwd_apply: bad args");
  PASE_LAUNCH((out_bwd_apply_kernel), blocks_for(rows * C, 256), 256, 0, (cudaStream_t)stream, 
      g, y, mean, invstd, scale, S1, S2, 1.0 / count, use_stats, rows, C);
  PASE_LAUNCH_CHECK("pase_out_bwd_apply");
  return PASE_OK;
}

int pase_nct_to_ntc(const float* src, float* dst, int N, int C, int T, long dst_row_stride,
                    void* stream) {
  PASE_CHECK_ARG(src && dst && N > 0 && C > 0 && T > 0, "pase_nct_to_ntc: bad args");
  dim3 grid((T + 31) / 32, (C + 31) / 32, N), block(32, 8);
  nct_to_ntc_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(src, dst, C, T, dst_row_stride);
  PASE_LAUNCH_CHECK("pase_nct_to_ntc");
  return PASE_OK;
}

int pase_ntc_to_nct(const float* src, long src_row_stride, float* dst, int N, int C, int T,
                    void* stream) {
  PASE_CHECK_ARG(src && dst && N > 0 && C > 0 && T > 0, "pase_ntc_to_nct: bad args");
  dim3 grid((T + 31) / 32, (C + 31) / 32, N), block(32, 8);
  ntc_to_nct_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(src, src_row_stride, dst, C, T);
  PASE_LAUNCH_CHECK("pase_ntc_to_nct");
  return PASE_OK;
}

int pase_axpy(const float* x, float* y, long n, float a, void* stream) {
  PASE_CHECK_ARG(x && y && n > 0, "pase_axpy: bad args");
  axpy_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, n, a);
  PASE_LAUNCH_CHECK("pase_axpy");
  return PASE_OK;
}

int pase_scale_dev(float* x, long n, const float* dev_scalar, float host_coef, void* stream) {
  PASE_CHECK_ARG(x && n > 0, "pase_scale_dev: bad args");
  scale_dev_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n, dev_scalar,
                                                                        host_coef);
  PASE_LAUNCH_CHECK("pase_scale_dev");
  return PASE_OK;
}

// ---- packed variable-length backward ------------------------------------------------------
static int bn_bwd_var_check(const char* fn, const void* y, int y_bf16, const int* tab, int nseg,
                            int max_T, int C, const void* srcA, int a_bf16, long a_row_stride,
                            const float* srcB, long b_row_stride, const float* pool,
                            long pool_row_stride) {
  PASE_CHECK_ARG(y && tab && srcA, "%s: null pointer", fn);
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && max_T > 0 && C > 0 && (C % 4) == 0 && C <= 4096,
                 "%s: nseg=%d max_T=%d C=%d", fn, nseg, max_T, C);
  PASE_CHECK_ARG(!a_bf16 || y_bf16, "%s: bf16 srcA needs bf16 y", fn);
  PASE_CHECK_QUAD(fn, y, y_bf16 ? 2 : 4, "y");
  PASE_CHECK_QUAD(fn, srcA, a_bf16 ? 2 : 4, "srcA");
  PASE_CHECK_STRIDE(fn, a_row_stride, "a_row_stride");
  PASE_CHECK_ARG(a_row_stride >= C, "%s: a_row_stride < C", fn);
  if (srcB) {
    PASE_CHECK_QUAD(fn, srcB, 4, "srcB");
    PASE_CHECK_STRIDE(fn, b_row_stride, "b_row_stride");
  }
  if (pool) {
    PASE_CHECK_QUAD(fn, pool, 4, "pool");
    PASE_CHECK_STRIDE(fn, pool_row_stride, "pool_row_stride");
  }
  return PASE_OK;
}

int pase_bn_prelu_bwd_reduce_var(const void* y, int y_bf16, const int* tab, int nseg, int max_T,
                                 int C, const float* mean, const float* invstd,
                                 const float* scale, const float* shift, const float* alpha,
                                 const void* srcA, int a_bf16, long a_row_stride, int padL,
                                 int padR, const float* srcB, long b_row_stride, int b_shift,
                                 const float* pool, long pool_row_stride, double* S1, double* S2,
                                 double* dalpha, float* amax, void* stream) {
  const char* fn = "pase_bn_prelu_bwd_reduce_var";
  PASE_CHECK_ARG(mean && invstd && scale && shift && alpha && S1 && S2 && dalpha,
                 "%s: null pointer", fn);
  const int rc = bn_bwd_var_check(fn, y, y_bf16, tab, nseg, max_T, C, srcA, a_bf16,
                                  a_row_stride, srcB, b_row_stride, pool, pool_row_stride);
  if (rc != PASE_OK) return rc;
  const long items = (long)(C / 4) * ((max_T + RUN - 1) / RUN);
  dim3 grid((unsigned)((items + THREADS - 1) / THREADS), nseg);
  const size_t sm = 3 * C * sizeof(double) + 2 * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_REDV(YT, GT)                                                                     \
  do {                                                                                        \
    if (sm > 48 * 1024)                                                                       \
      cudaFuncSetAttribute(bn_prelu_bwd_reduce_var_kernel<YT, GT>,                            \
                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);             \
    PASE_LAUNCH((bn_prelu_bwd_reduce_var_kernel<YT, GT>), grid, THREADS, sm, st,              \
                reinterpret_cast<const YT*>(y), tab, C, mean, invstd, scale, shift, alpha,    \
                srcA, a_row_stride, padL, padR, srcB, b_row_stride, b_shift, pool,            \
                pool_row_stride, S1, S2, dalpha, amax);                                       \
  } while (0)
  if (y_bf16) {
    if (a_bf16) PASE_REDV(__nv_bfloat16, __nv_bfloat16);
    else PASE_REDV(__nv_bfloat16, float);
  } else {
    PASE_REDV(float, float);
  }
#undef PASE_REDV
  PASE_LAUNCH_CHECK(fn);
  return PASE_OK;
}

// pase_bn_prelu_bwd_apply_src_var (mean, S1, S2 NULL: eval mode) and its train-mode form
static int bn_apply_src_var(const char* fn, const void* y, int y_bf16, const int* tab, int nseg,
                            int max_span, int C, const float* mean, const float* invstd,
                            const float* gamma, const float* scale, const float* shift,
                            const float* alpha, const double* S1, const double* S2, double count,
                            const void* srcA, int a_bf16, long a_row_stride, int padL, int padR,
                            const float* srcB, long b_row_stride, int b_shift, const float* pool,
                            long pool_row_stride, void* dst, void* dst_lo, int dst_fmt, int lead,
                            double* dbias_acc, const float* amax, float* scale_out,
                            void* stream) {
  const bool train = S1 != nullptr;
  PASE_CHECK_ARG(invstd && scale && shift && alpha && dst && lead >= 0, "%s: null pointer / lead",
                 fn);
  const int rc = bn_bwd_var_check(fn, y, y_bf16, tab, nseg, max_span, C, srcA, a_bf16,
                                  a_row_stride, srcB, b_row_stride, pool, pool_row_stride);
  if (rc != PASE_OK) return rc;
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2, "%s: bad dst_fmt %d", fn, dst_fmt);
  PASE_CHECK_ARG(dst_fmt != PASE_FMT_F16X2 || (dst_lo && amax && scale_out && !y_bf16),
                 "%s: the fp16-pair format needs dst_lo, amax, scale_out and fp32 y", fn);
  PASE_CHECK_ARG((dst_fmt == PASE_FMT_BF16) == (y_bf16 != 0),
                 "%s: bf16 y goes with bf16 dst (and only with it)", fn);
  PASE_CHECK_QUAD(fn, dst, dst_fmt == PASE_FMT_F32 ? 4 : 2, "dst");
  // runs of the T frames + zero runs of [T, span) and the lead: at most this many per row
  const long items = (long)(C / 4) * ((max_span + RUN - 1) / RUN + (lead + RUN - 1) / RUN + 1);
  dim3 grid((unsigned)((items + THREADS - 1) / THREADS), nseg);
  const size_t sm = C * sizeof(double) + sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_APSV(YT, GT, DF)                                                                  \
  do {                                                                                         \
    if (train)                                                                                 \
      PASE_LAUNCH((bn_prelu_bwd_apply_src_var_train_kernel<YT, GT, DF>), grid, THREADS, sm, st, \
                  reinterpret_cast<const YT*>(y), tab, C, mean, invstd, gamma, scale, shift,    \
                  alpha, S1, S2, 1.0 / count, srcA, a_row_stride, padL, padR, srcB,             \
                  b_row_stride, b_shift, pool, pool_row_stride, dst, dst_lo, lead, dbias_acc,   \
                  amax, scale_out);                                                            \
    else                                                                                       \
      PASE_LAUNCH((bn_prelu_bwd_apply_src_var_kernel<YT, GT, DF>), grid, THREADS, sm, st,      \
                  reinterpret_cast<const YT*>(y), tab, C, invstd, gamma, scale, shift, alpha,   \
                  srcA, a_row_stride, padL, padR, srcB, b_row_stride, b_shift, pool,            \
                  pool_row_stride, dst, dst_lo, lead, dbias_acc, amax, scale_out);             \
  } while (0)
  if (dst_fmt == PASE_FMT_BF16) {
    if (a_bf16) PASE_APSV(__nv_bfloat16, __nv_bfloat16, PASE_FMT_BF16);
    else PASE_APSV(__nv_bfloat16, float, PASE_FMT_BF16);
  } else if (dst_fmt == PASE_FMT_F16X2) {
    PASE_APSV(float, float, PASE_FMT_F16X2);
  } else {
    PASE_APSV(float, float, PASE_FMT_F32);
  }
#undef PASE_APSV
  PASE_LAUNCH_CHECK(fn);
  return PASE_OK;
}

int pase_bn_prelu_bwd_apply_src_var(const void* y, int y_bf16, const int* tab, int nseg,
                                    int max_span, int C, const float* invstd, const float* gamma,
                                    const float* scale, const float* shift, const float* alpha,
                                    const void* srcA, int a_bf16, long a_row_stride, int padL,
                                    int padR, const float* srcB, long b_row_stride, int b_shift,
                                    const float* pool, long pool_row_stride, void* dst,
                                    void* dst_lo, int dst_fmt, int lead, double* dbias_acc,
                                    const float* amax, float* scale_out, void* stream) {
  return bn_apply_src_var("pase_bn_prelu_bwd_apply_src_var", y, y_bf16, tab, nseg, max_span, C,
                          nullptr, invstd, gamma, scale, shift, alpha, nullptr, nullptr, 1.0,
                          srcA, a_bf16, a_row_stride, padL, padR, srcB, b_row_stride, b_shift,
                          pool, pool_row_stride, dst, dst_lo, dst_fmt, lead, dbias_acc, amax,
                          scale_out, stream);
}

int pase_bn_prelu_bwd_apply_src_var_train(
    const void* y, int y_bf16, const int* tab, int nseg, int max_span, int C, const float* mean,
    const float* invstd, const float* gamma, const float* scale, const float* shift,
    const float* alpha, const double* S1, const double* S2, double count, const void* srcA,
    int a_bf16, long a_row_stride, int padL, int padR, const float* srcB, long b_row_stride,
    int b_shift, const float* pool, long pool_row_stride, void* dst, void* dst_lo, int dst_fmt,
    int lead, double* dbias_acc, const float* amax, float* scale_out, void* stream) {
  const char* fn = "pase_bn_prelu_bwd_apply_src_var_train";
  PASE_CHECK_ARG(mean && S1 && S2 && count >= 1.0, "%s: null statistics or count %g < 1", fn,
                 count);
  return bn_apply_src_var(fn, y, y_bf16, tab, nseg, max_span, C, mean, invstd, gamma, scale, shift,
                          alpha, S1, S2, count, srcA, a_bf16, a_row_stride, padL, padR, srcB,
                          b_row_stride, b_shift, pool, pool_row_stride, dst, dst_lo, dst_fmt,
                          lead, dbias_acc, amax, scale_out, stream);
}

int pase_out_bwd_reduce_var(const float* dout, const int* tab, int nseg, int max_T, int C,
                            const float* y, const float* mean, const float* invstd, float* g_ntc,
                            double* S1, double* S2, void* stream) {
  PASE_CHECK_ARG(dout && tab && y && mean && invstd && g_ntc && S1 && S2,
                 "pase_out_bwd_reduce_var: null pointer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && max_T > 0 && C > 0,
                 "pase_out_bwd_reduce_var: nseg=%d max_T=%d C=%d", nseg, max_T, C);
  dim3 grid((max_T + 31) / 32, (C + 31) / 32, nseg), block(32, 8);
  PASE_LAUNCH((out_bwd_reduce_var_kernel), grid, block, 0, (cudaStream_t)stream, dout, tab, y,
              mean, invstd, C, g_ntc, S1, S2);
  PASE_LAUNCH_CHECK("pase_out_bwd_reduce_var");
  return PASE_OK;
}

int pase_out_bwd_gather_var(const float* dout, const int* tab, int nseg, int max_T, int C,
                            float* g_ntc, void* stream) {
  PASE_CHECK_ARG(dout && tab && g_ntc && nseg > 0 && nseg <= 65535 && max_T > 0 && C > 0,
                 "pase_out_bwd_gather_var: bad args");
  const long total = (long)max_T * C;
  long bx = (total + 255) / 256;
  if (bx > 1024) bx = 1024;
  PASE_LAUNCH((out_bwd_gather_var_kernel), dim3((unsigned)bx, nseg), 256, 0, (cudaStream_t)stream,
              dout, tab, C, g_ntc);
  PASE_LAUNCH_CHECK("pase_out_bwd_gather_var");
  return PASE_OK;
}

int pase_out_bwd_gather_crop(const float* dout, long ld, long col0, int T, int c0, int cn, int C,
                             float* g_ntc, void* stream) {
  PASE_CHECK_ARG(dout && g_ntc && T > 0 && C > 0 && c0 >= 0 && cn > 0 && c0 + cn <= T &&
                     col0 >= 0 && col0 + cn <= ld,
                 "pase_out_bwd_gather_crop: bad args (T=%d crop %d+%d, col0=%ld ld=%ld)", T, c0,
                 cn, col0, ld);
  const long total = (long)T * C;
  long bx = (total + 255) / 256;
  if (bx > 1024) bx = 1024;
  PASE_LAUNCH((out_bwd_gather_crop_kernel), dim3((unsigned)bx), 256, 0, (cudaStream_t)stream, dout,
              ld, col0, T, c0, cn, C, g_ntc);
  PASE_LAUNCH_CHECK("pase_out_bwd_gather_crop");
  return PASE_OK;
}

}  // extern "C"
