// Padding, BatchNorm (batch statistics), PReLU and dense-skip pooling kernels.
// All HBM-bound: channel-last float4 accesses, one pass per tensor.
#include "common.cuh"
#include "bn_stream.cuh"
#include <cstdlib>

namespace {

constexpr int THREADS = 256;

// DF: operand format of the padded waveform (block 0's GEMM operand)
template <int DF>
__global__ void reflect_pad_wave_kernel(const float* __restrict__ x, void* __restrict__ dst_v,
                                        void* __restrict__ dst_lo_v, int T, int padL, int Tp,
                                        long pitch) {
  pdl_wait();
  const int n = blockIdx.y;
  for (int tau = blockIdx.x * blockDim.x + threadIdx.x; tau < Tp; tau += gridDim.x * blockDim.x) {
    const float v = x[(long)n * T + reflect_idx(tau - padL, T)];
    const long o = (long)n * pitch + tau;
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
//   reads (i.e. after rounding to bf16 in the bf16 format); the thread that writes the first
//   time step of a pooling window sums the whole window in time order, so each window mean
//   has one writer and comes out the same on every run.
template <typename YT, int DF, int RUN>
__global__ void __launch_bounds__(THREADS)
bn_prelu_pad_fwd_kernel(const YT* __restrict__ y, long y_ss, int T, int C,
                        const float* __restrict__ scale, const float* __restrict__ shift,
                        const float* __restrict__ alpha, void* __restrict__ dst_v, long d_ss,
                        long d_rs, int padL, int Tp, float* __restrict__ pool, long p_ss,
                        long p_rs, int pool_d, int pool_T, void* __restrict__ dst_lo_v) {
  pdl_wait();
  const int C4 = C >> 2;
  const int n = blockIdx.y;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int q = (int)(idx % C4);
  const long run = idx / C4;
  const long tau0 = run * RUN;
  if (tau0 >= Tp) return;
  const int c = q * 4;
  const float4 sc = ld4(scale + c), sh = ld4(shift + c), al = ld4(alpha + c);
  const YT* yn = y + (long)n * y_ss;
  const int pool_len = pool_d > 0 ? pool_T * pool_d : 0;
  const float inv_d = pool_d > 0 ? 1.f / (float)pool_d : 0.f;
  const int nvalid = (Tp - tau0) < RUN ? (int)(Tp - tau0) : RUN;
  float4 vals[RUN];
#pragma unroll
  for (int i = 0; i < RUN; ++i)
    if (i < nvalid) vals[i] = ld4t(yn + (long)reflect_idx((int)tau0 + i - padL, T) * C + c);
#pragma unroll
  for (int i = 0; i < RUN; ++i) {
    if (i >= nvalid) break;
    const long tau = tau0 + i;
    const int tr = (int)tau - padL;
    const float4 v = vals[i];
    float4 a;
    a.x = prelu1(fmaf(v.x, sc.x, sh.x), al.x);
    a.y = prelu1(fmaf(v.y, sc.y, sh.y), al.y);
    a.z = prelu1(fmaf(v.z, sc.z, sh.z), al.z);
    a.w = prelu1(fmaf(v.w, sc.w, sh.w), al.w);
    const long o = (long)n * d_ss + tau * d_rs + c;
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
    if (tr >= 0 && tr < pool_len && tr % pool_d == 0) {
      float4 ps = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < pool_d; ++k) {
        const float4 w = ld4t(yn + (long)(tr + k) * C + c);
        float4 b;
        b.x = prelu1(fmaf(w.x, sc.x, sh.x), al.x);
        b.y = prelu1(fmaf(w.y, sc.y, sh.y), al.y);
        b.z = prelu1(fmaf(w.z, sc.z, sh.z), al.z);
        b.w = prelu1(fmaf(w.w, sc.w, sh.w), al.w);
        if constexpr (DF == PASE_FMT_BF16) b = rt4t(static_cast<const __nv_bfloat16*>(nullptr), b);
        ps.x += b.x; ps.y += b.y; ps.z += b.z; ps.w += b.w;
      }
      float* pp = pool + (long)n * p_ss + (long)(tr / pool_d) * p_rs + c;
      atomicAdd(pp + 0, ps.x * inv_d);
      atomicAdd(pp + 1, ps.y * inv_d);
      atomicAdd(pp + 2, ps.z * inv_d);
      atomicAdd(pp + 3, ps.w * inv_d);
    }
  }
}

// ---- backward pass 1: du + reductions ----
// (BwdSrc: bn_stream.cuh)

// The gradient reaching this block's output for one run of RUN time steps (t0 ..) of the
// channel quad at c: source A (the next layer's padded input gradient, reflect halo folded
// back at the two sequence ends), the optional shifted source B (QRNN) and the broadcast of
// the mean-pooled dense-skip gradient.  Straight-line loads first (no branch between a load
// and the next one, so all DRAM requests of the run are in flight together).
template <typename GT, int RUN>
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
template <typename YT, typename GT, int RUN>
__global__ void __launch_bounds__(THREADS, RUN <= 4 ? 2 : 1)
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
    load_grad_run<GT, RUN>(s, n, T, t0, nvalid, c, gs);
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
template <typename YT, int DF, int RUN>
__global__ void __launch_bounds__(THREADS, RUN <= 4 ? 3 : 2)
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
template <typename YT, typename GT, int DF, int RUN>
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
      load_grad_run<GT, RUN>(s, n, T, t0, nvalid, c, gs);
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
__global__ void out_affine_nct_kernel(const float* __restrict__ y, const float* __restrict__ scale,
                                      const float* __restrict__ shift, float* __restrict__ out,
                                      float* __restrict__ out_ntc, int T, int C) {
  pdl_wait();
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) {
      const float v = fmaf(y[((long)n * T + t) * C + c], scale[c], shift[c]);
      tile[i][threadIdx.x] = v;
      if (out_ntc) out_ntc[((long)n * T + t) * C + c] = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (t < T && c < C) out[((long)n * C + c) * T + t] = tile[threadIdx.x][i];
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
  __shared__ float tile[32][33];
  __shared__ double r1[32], r2[32];   // fp64: order-independent to fp32 precision
  const int n = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  if (threadIdx.y == 0) { r1[threadIdx.x] = 0.0; r2[threadIdx.x] = 0.0; }
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (dout && t < T && c < C) ? dout[((long)n * C + c) * T + t] : 0.f;
  }
  __syncthreads();
  float a1 = 0.f, a2 = 0.f;
  const int c = c0 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i;
    if (t < T && c < C) {
      const long o = ((long)n * T + t) * C + c;
      float g = tile[threadIdx.x][i];
      if (dout_ntc) g += dout_ntc[o];
      g_ntc[o] = g;
      const float xh = (y[o] - mean[c]) * invstd[c];
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

// time steps per thread of the BatchNorm / PReLU passes: 8 (default; measured 3.31 vs 3.42
// ms/step against 4 steps per thread with 2-3 resident blocks per SM: loads in flight per
// thread matter more than occupancy here); PASE_B200_BN_RUN=4 selects the other variant
inline int bn_run() {
  static int r = 0;
  if (r == 0) {
    const char* e = getenv("PASE_B200_BN_RUN");
    r = (e && atoi(e) == 4) ? 4 : 8;
  }
  return r;
}

inline unsigned blocks_for(long total, int threads, int cap_mult = 8) {
  long b = (total + threads - 1) / threads;
  long cap = (long)pase_num_sms() * cap_mult;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
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
  cudaStream_t st = (cudaStream_t)stream;
  if (dst_fmt == PASE_FMT_F32)
    PASE_LAUNCH((reflect_pad_wave_kernel<PASE_FMT_F32>), grid, 256, 0, st, x, dst, dst_lo, T, padL, Tp, pitch);
  else if (dst_fmt == PASE_FMT_BF16)
    PASE_LAUNCH((reflect_pad_wave_kernel<PASE_FMT_BF16>), grid, 256, 0, st, x, dst, dst_lo, T, padL, Tp, pitch);
  else
    PASE_LAUNCH((reflect_pad_wave_kernel<PASE_FMT_F16X2>), grid, 256, 0, st, x, dst, dst_lo, T, padL, Tp, pitch);
  PASE_LAUNCH_CHECK("pase_reflect_pad_wave");
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
  PASE_CHECK_ARG((dst_row_stride % 4) == 0 && (dst_sample_stride % 4) == 0 &&
                     (y_sample_stride % 4) == 0 && aligned16(y) && aligned16(dst),
                 "pase_bn_prelu_pad_fwd: strides/pointers must be 4-element aligned");
  PASE_CHECK_ARG(dst_fmt >= 0 && dst_fmt <= 2 && (dst_fmt != PASE_FMT_F16X2 || dst_lo),
                 "pase_bn_prelu_pad_fwd: bad dst_fmt %d / missing lo", dst_fmt);
  if (pool == nullptr) pool_d = 0;
  const int Tp = T + padL + padR;
  const int RUN = bn_run();
  const long threads = (long)(C / 4) * ((Tp + RUN - 1) / RUN);
  dim3 grid((unsigned)((threads + THREADS - 1) / THREADS), N);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_FWD_R(YT, DF, RV)                                                                 \
  PASE_LAUNCH((bn_prelu_pad_fwd_kernel<YT, DF, RV>), grid, THREADS, 0, st,                                \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, scale, shift, alpha, dst,         \
      dst_sample_stride, dst_row_stride, padL, Tp, pool, pool_sample_stride, pool_row_stride, \
      pool_d, pool_T, dst_lo)
#define PASE_FWD(YT, DF) do { if (RUN == 8) PASE_FWD_R(YT, DF, 8); else PASE_FWD_R(YT, DF, 4); } while (0)
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
#undef PASE_FWD_R
  PASE_LAUNCH_CHECK("pase_bn_prelu_pad_fwd");
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
  BwdSrc s{srcA, a_sample_stride, a_row_stride, padL, padR, srcB, b_sample_stride, b_row_stride,
           b_shift, pool, pool_sample_stride, pool_row_stride, pool ? pool_d : 0, pool_T};
  if (dst == nullptr) {                    // sums only: persistent staged kernel when it fits
    BnStreamArgs sa{};
    sa.y = y; sa.y_bf16 = y_bf16; sa.y_ss = y_sample_stride; sa.N = N; sa.T = T; sa.C = C;
    sa.mean = mean; sa.invstd = invstd; sa.scale = scale; sa.shift = shift; sa.alpha = alpha;
    sa.s = s; sa.a_bf16 = a_bf16; sa.S1 = S1; sa.S2 = S2; sa.dalpha = dalpha; sa.amax = amax;
    if (pase_bn_stream_ok(sa)) return pase_bn_stream_reduce(sa, (cudaStream_t)stream);
  }
  const int RUN = bn_run();
  const long threads = (long)(C / 4) * ((T + RUN - 1) / RUN);
  long gx = (threads + THREADS - 1) / THREADS;
  if ((THREADS % (C / 4)) == 0) {          // stride keeps the channel quad: cap the grid
    long cap = ((RUN == 8 ? 8L : 16L) * pase_num_sms() + N - 1) / N;
    if (cap < 1) cap = 1;
    if (gx > cap) gx = cap;
  }
  dim3 grid((unsigned)gx, N);
  const size_t sm = 3 * C * sizeof(double) + 2 * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_RED_R(YT, GT, RV)                                                               \
  bn_prelu_bwd_reduce_kernel<YT, GT, RV><<<grid, THREADS, sm, st>>>(                         \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, mean, invstd, scale, shift,     \
      alpha, s, reinterpret_cast<YT*>(dst), dst_sample_stride, S1, S2, dalpha, amax)
#define PASE_RED(YT, GT) do { if (RUN == 8) PASE_RED_R(YT, GT, 8); else PASE_RED_R(YT, GT, 4); } while (0)
  if (y_bf16) {
    if (a_bf16) PASE_RED(__nv_bfloat16, __nv_bfloat16);
    else PASE_RED(__nv_bfloat16, float);
  } else {
    if (a_bf16) PASE_RED(float, __nv_bfloat16);
    else PASE_RED(float, float);
  }
#undef PASE_RED
#undef PASE_RED_R
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
  const int RUN = bn_run();
  const long threads = (long)(C / 4) * ((T + RUN - 1) / RUN);
  long gx = (threads + THREADS - 1) / THREADS;
  if ((THREADS % (C / 4)) == 0) {
    long cap = ((RUN == 8 ? 8L : 16L) * pase_num_sms() + N - 1) / N;
    if (cap < 1) cap = 1;
    if (gx > cap) gx = cap;
  }
  dim3 grid((unsigned)gx, N);
  const size_t sm = C * sizeof(double) + sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_APP_R(YT, DF, RV)                                                                \
  bn_prelu_bwd_apply_kernel<YT, DF, RV><<<grid, THREADS, sm, st>>>(                           \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, mean, invstd, gamma, S1, S2,     \
      1.0 / count, reinterpret_cast<const YT*>(du), dst, dst_sample_stride, dbias_acc,        \
      dst_lo, amax, scale_out)
#define PASE_APP(YT, DF) do { if (RUN == 8) PASE_APP_R(YT, DF, 8); else PASE_APP_R(YT, DF, 4); } while (0)
  if (dst_fmt == PASE_FMT_BF16) PASE_APP(__nv_bfloat16, PASE_FMT_BF16);
  else if (dst_fmt == PASE_FMT_F16X2) PASE_APP(float, PASE_FMT_F16X2);
  else PASE_APP(float, PASE_FMT_F32);
#undef PASE_APP
#undef PASE_APP_R
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
  BwdSrc s{srcA, a_sample_stride, a_row_stride, padL, padR, srcB, b_sample_stride, b_row_stride,
           b_shift, pool, pool_sample_stride, pool_row_stride, pool ? pool_d : 0, pool_T};
  {
    BnStreamArgs sa{};
    sa.y = y; sa.y_bf16 = y_bf16; sa.y_ss = y_sample_stride; sa.N = N; sa.T = T; sa.C = C;
    sa.mean = mean; sa.invstd = invstd; sa.gamma = gamma; sa.scale = scale; sa.shift = shift;
    sa.alpha = alpha; sa.s = s; sa.a_bf16 = a_bf16; sa.S1in = S1; sa.S2in = S2;
    sa.inv_count = 1.0 / count; sa.dst = dst; sa.dst_lo = dst_lo; sa.dst_fmt = dst_fmt;
    sa.d_ss = dst_sample_stride; sa.dbias = dbias_acc; sa.amax = const_cast<float*>(amax); sa.scale_out = scale_out;
    if (pase_bn_stream_ok(sa) && (dst_sample_stride % 8) == 0 && aligned16(dst) &&
        (dst_lo == nullptr || aligned16(dst_lo)))
      return pase_bn_stream_apply(sa, (cudaStream_t)stream);
  }
  const int RUN = bn_run();
  const long threads = (long)(C / 4) * ((T + RUN - 1) / RUN);
  long gx = (threads + THREADS - 1) / THREADS;
  if ((THREADS % (C / 4)) == 0) {
    long cap = ((RUN == 8 ? 8L : 16L) * pase_num_sms() + N - 1) / N;
    if (cap < 1) cap = 1;
    if (gx > cap) gx = cap;
  }
  dim3 grid((unsigned)gx, N);
  const size_t sm = C * sizeof(double) + sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_APS_R(YT, GT, DF, RV)                                                             \
  bn_prelu_bwd_apply_src_kernel<YT, GT, DF, RV><<<grid, THREADS, sm, st>>>(                    \
      reinterpret_cast<const YT*>(y), y_sample_stride, T, C, mean, invstd, gamma, scale, shift, \
      alpha, S1, S2, 1.0 / count, s, dst, dst_sample_stride, dbias_acc, dst_lo, amax, scale_out)
#define PASE_APS(YT, GT, DF) do { if (RUN == 8) PASE_APS_R(YT, GT, DF, 8); else PASE_APS_R(YT, GT, DF, 4); } while (0)
  if (dst_fmt == PASE_FMT_BF16) {
    if (a_bf16) PASE_APS(__nv_bfloat16, __nv_bfloat16, PASE_FMT_BF16);
    else PASE_APS(__nv_bfloat16, float, PASE_FMT_BF16);
  } else if (dst_fmt == PASE_FMT_F16X2) {
    PASE_APS(float, float, PASE_FMT_F16X2);
  } else {
    PASE_APS(float, float, PASE_FMT_F32);
  }
#undef PASE_APS
#undef PASE_APS_R
  PASE_LAUNCH_CHECK("pase_bn_prelu_bwd_apply_src");
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

int pase_out_bwd_reduce(const float* dout, const float* dout_ntc, const float* y,
                        const float* mean, const float* invstd, int N, int T, int C, float* g_ntc,
                        double* S1, double* S2, void* stream) {
  PASE_CHECK_ARG((dout || dout_ntc) && y && mean && invstd && g_ntc && S1 && S2,
                 "pase_out_bwd_reduce: null pointer");
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

}  // extern "C"
