// BatchNorm/PReLU backward passes as persistent, shared-memory staged streaming kernels.
//
// The register-resident kernels of act.cu keep one run of loads in flight per thread; at
// ~200 registers that is one 256-thread block per SM, and the passes over the 26 MB mid-layer
// tensors run at 2.5 TB/s (latency-bound: load, reduce, exit, next block).  Here every block
// is persistent and streams (time-tile x C) slabs of y and of the gradient source through a
// 3-stage shared-memory ring filled by cp.async.bulk (the TMA engine; completion on an
// mbarrier): the bytes in flight per SM (2 blocks x 2 stages x 32 KB) no longer depend on
// registers, and the per-block reductions happen once per SM instead of once per 70 KB.
#include "bn_stream.cuh"
#include <cstdlib>

namespace {

constexpr int THREADS = 256;
// tile configuration: TE = TT * C elements per tensor per stage, NS stages
//   <4096, 3>: 32 KB (fp32 y + g) per stage, 2 in flight per block
//   <2048, 6>: 16 KB per stage, 5 in flight per block (same shared memory, deeper queue)

__device__ __forceinline__ uint32_t s_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void bar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool bar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(s_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!bar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();          // a lost bulk copy must not hang the box
  }
}
// global -> shared bulk copy (16-byte aligned, size a multiple of 16), completion on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(s_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(s_u32(bar))
      : "memory");
}

struct Geo {
  int tps;            // tiles per sample
  long total;         // N * tps
  int TT;
};

template <int TE_, int NS_>
struct TileCfg {
  static constexpr int TE = TE_, NS = NS_;
  static constexpr int ITEMS = TE_ / 4 / THREADS;   // float4 quads per thread per tile
};

// One tile of y and of gradient source A into stage `st` (called by one thread).
template <typename YT, typename GT, int TILE_ELEMS>
__device__ __forceinline__ void issue_tile(const BnStreamArgs& a, const Geo& g, long tile,
                                           uint8_t* stage, uint64_t* bar) {
  const int n = (int)(tile / g.tps);
  const int t0 = (int)(tile % g.tps) * g.TT;
  const int rows = (a.T - t0) < g.TT ? (a.T - t0) : g.TT;
  const int C = a.C;
  const uint32_t by = (uint32_t)rows * C * sizeof(YT), bg = (uint32_t)rows * C * sizeof(GT);
  bar_expect_tx(bar, by + bg);
  const YT* ysrc = reinterpret_cast<const YT*>(a.y) + (long)n * a.y_ss + (long)t0 * C;
  bulk_g2s(stage, ysrc, by, bar);
  uint8_t* sg = stage + TILE_ELEMS * sizeof(YT);
  const GT* gsrc = reinterpret_cast<const GT*>(a.s.A) + (long)n * a.s.a_ss +
                   (long)(t0 + a.s.padL) * a.s.a_rs;
  if (a.s.a_rs == C) {
    bulk_g2s(sg, gsrc, bg, bar);
  } else {
    const uint32_t rb = (uint32_t)C * sizeof(GT);
    for (int r = 0; r < rows; ++r) bulk_g2s(sg + (size_t)r * rb, gsrc + (long)r * a.s.a_rs, rb, bar);
  }
}

// APPLY = false: pass 1 (S1, S2, dalpha, amax).  APPLY = true: pass 2 (dy in format DF, db).
template <typename YT, typename GT, int DF, bool APPLY, typename TC>
__global__ void __launch_bounds__(THREADS, 2)
bn_bwd_stream_kernel(const BnStreamArgs a, const Geo g) {
  constexpr int TILE_ELEMS = TC::TE, STAGES = TC::NS, ITEMS = TC::ITEMS;
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int STAGE_BYTES = TILE_ELEMS * (sizeof(YT) + sizeof(GT));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  // block sums in fp64 ([3C] or [C]): the order of the threads' additions then only moves
  // bits below fp32 precision (run-to-run identical statistics); maxima ([2] or [1]) in fp32
  double* red = reinterpret_cast<double*>(bars + STAGES);
  const int C = a.C, C4 = C >> 2, T = a.T;
  float* redm = reinterpret_cast<float*>(red + (APPLY ? C : 3 * C));
  const int tid = threadIdx.x;
  const int q = tid % C4, r0 = tid / C4, rstep = THREADS / C4;
  const int c = q * 4;
  for (int i = tid; i < (APPLY ? C : 3 * C); i += THREADS) red[i] = 0.0;
  if (tid < 2) redm[tid] = 0.f;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) bar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  // prologue: fill the ring
  const long first = blockIdx.x, stride = gridDim.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      const long tile = first + (long)s * stride;
      if (tile < g.total) issue_tile<YT, GT, TILE_ELEMS>(a, g, tile, smem + s * STAGE_BYTES, &bars[s]);
    }
  }
  float gs_scale = 1.f;
  if constexpr (APPLY && DF == PASE_FMT_F16X2) {
    const float mdu = a.amax[0], mxh = a.amax[1];
    float b = 0.f;
    for (int i = tid; i < C; i += THREADS) {
      const float gi = fabsf((a.gamma ? a.gamma[i] : 1.f) * a.invstd[i]);
      const float m1 = fabsf((float)(a.S1in[i] * a.inv_count));
      const float m2 = fabsf((float)(a.S2in[i] * a.inv_count));
      b = fmaxf(b, gi * (mdu + m1 + mxh * m2));
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, off));
    if ((tid & 31) == 0) atomic_max_pos(&redm[0], b);
    __syncthreads();
    gs_scale = f16_grad_scale(redm[0] * 1.0001f);
    if (blockIdx.x == 0 && tid == 0) {
      a.scale_out[0] = 1.f / gs_scale;
      a.scale_out[1] = gs_scale;
    }
  }
  // per-thread channel constants (the channel quad is fixed for the whole kernel)
  float scv[4], shv[4], alv[4], muv[4], isv[4], m1[4], m2[4], gi[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    scv[k] = a.scale[c + k];
    shv[k] = a.shift[c + k];
    alv[k] = a.alpha[c + k];
    muv[k] = a.mean[c + k];
    isv[k] = a.invstd[c + k];
    if constexpr (APPLY) {
      m1[k] = (float)(a.S1in[c + k] * a.inv_count);
      m2[k] = (float)(a.S2in[c + k] * a.inv_count);
      gi[k] = (a.gamma ? a.gamma[c + k] : 1.f) * isv[k];
    }
  }
  float a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0}, a3[4] = {0, 0, 0, 0};
  float mx_du = 0.f, mx_xh = 0.f;
  const bool has_pool = a.s.P != nullptr && a.s.pool_d > 0;
  const int pool_len = has_pool ? a.s.pool_T * a.s.pool_d : 0;
  const float inv_d = has_pool ? 1.f / (float)a.s.pool_d : 0.f;
  // pooled dense-skip gradient of the NEXT tile, fetched one tile ahead (L2 latency hidden
  // behind the current tile's work)
  float4 pv[ITEMS];
  auto fetch_pool = [&](long tile) {
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) pv[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!has_pool || tile >= g.total) return;
    const int n = (int)(tile / g.tps);
    const int t0 = (int)(tile % g.tps) * g.TT;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int t = t0 + r0 + k * rstep;
      if (t < pool_len)
        pv[k] = *reinterpret_cast<const float4*>(a.s.P + (long)n * a.s.p_ss +
                                                 (long)(t / a.s.pool_d) * a.s.p_rs + c);
    }
  };
  fetch_pool(first);
  int stage = 0;
  uint32_t phase = 0;
  for (long tile = first; tile < g.total; tile += stride) {
    const int n = (int)(tile / g.tps);
    const int t0 = (int)(tile % g.tps) * g.TT;
    const int rows = (T - t0) < g.TT ? (T - t0) : g.TT;
    float4 pcur[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) pcur[k] = pv[k];
    bar_wait(&bars[stage], phase);
    const YT* sy = reinterpret_cast<const YT*>(smem + stage * STAGE_BYTES);
    const GT* sg = reinterpret_cast<const GT*>(smem + stage * STAGE_BYTES + TILE_ELEMS * sizeof(YT));
    float4 vs[ITEMS], gs[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int r = r0 + k * rstep;
      const int rr = r < rows ? r : 0;
      vs[k] = ld4t(sy + rr * C + c);
      gs[k] = ld4t(sg + rr * C + c);
    }
    fetch_pool(tile + stride);
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      gs[k].x += pcur[k].x * inv_d; gs[k].y += pcur[k].y * inv_d;
      gs[k].z += pcur[k].z * inv_d; gs[k].w += pcur[k].w * inv_d;
    }
    // rare: reflect-pad fold-back at the two sequence ends, second shifted source (QRNN)
    const bool edge = (a.s.padL > 0 && t0 <= a.s.padL) ||
                      (a.s.padR > 0 && t0 + g.TT >= T - 1 - a.s.padR);
    if (edge || a.s.B != nullptr) {
      const GT* an = reinterpret_cast<const GT*>(a.s.A) + (long)n * a.s.a_ss + c;
#pragma unroll
      for (int k = 0; k < ITEMS; ++k) {
        const int r = r0 + k * rstep;
        if (r >= rows) continue;
        const int t = t0 + r;
        float4 gg = gs[k];
        auto add4 = [&](float4 v) { gg.x += v.x; gg.y += v.y; gg.z += v.z; gg.w += v.w; };
        if (a.s.padL > 0 && t >= 1 && t <= a.s.padL) add4(ld4t(an + (long)(a.s.padL - t) * a.s.a_rs));
        if (a.s.padR > 0 && t <= T - 2 && t >= T - 1 - a.s.padR)
          add4(ld4t(an + (long)(a.s.padL + 2 * (T - 1) - t) * a.s.a_rs));
        if (a.s.B) {
          const int tb = t + a.s.b_shift;
          if (tb >= 0 && tb < T)
            add4(*reinterpret_cast<const float4*>(a.s.B + (long)n * a.s.b_ss +
                                                  (long)tb * a.s.b_rs + c));
        }
        gs[k] = gg;
      }
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int r = r0 + k * rstep;
      if (r >= rows) continue;
      const int t = t0 + r;
      const float vv[4] = {vs[k].x, vs[k].y, vs[k].z, vs[k].w};
      const float gg[4] = {gs[k].x, gs[k].y, gs[k].z, gs[k].w};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float u = fmaf(vv[j], scv[j], shv[j]);
        const bool pos = u > 0.f;
        const float du = pos ? gg[j] : alv[j] * gg[j];
        const float xh = (vv[j] - muv[j]) * isv[j];
        if constexpr (APPLY) {
          o[j] = gi[j] * (du - m1[j] - xh * m2[j]);
          a1[j] += o[j];
        } else {
          a3[j] += pos ? 0.f : u * gg[j];
          a1[j] += du;
          a2[j] += du * xh;
          mx_du = fmaxf(mx_du, fabsf(du));
          mx_xh = fmaxf(mx_xh, fabsf(xh));
        }
      }
      if constexpr (APPLY) {
        const long off = (long)n * a.d_ss + (long)t * C + c;
        if constexpr (DF == PASE_FMT_F32) {
          *reinterpret_cast<float4*>(reinterpret_cast<float*>(a.dst) + off) =
              make_float4(o[0], o[1], o[2], o[3]);
          if (a.dst_lo != nullptr)
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(a.dst_lo) + off) =
                make_float4(tf32_residual(o[0]), tf32_residual(o[1]), tf32_residual(o[2]),
                            tf32_residual(o[3]));
        } else if constexpr (DF == PASE_FMT_BF16) {
          st4t(reinterpret_cast<__nv_bfloat16*>(a.dst) + off, make_float4(o[0], o[1], o[2], o[3]));
        } else {
          st4_f16x2(reinterpret_cast<__half*>(a.dst) + off, reinterpret_cast<__half*>(a.dst_lo) + off,
                    make_float4(o[0] * gs_scale, o[1] * gs_scale, o[2] * gs_scale,
                                o[3] * gs_scale));
        }
      }
    }
    __syncthreads();                               // every thread is done with this stage
    if (tid == 0) {
      const long nxt = tile + (long)STAGES * stride;
      if (nxt < g.total) issue_tile<YT, GT, TILE_ELEMS>(a, g, nxt, smem + stage * STAGE_BYTES, &bars[stage]);
    }
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  // ---- block reduction: once per persistent block ----
  if constexpr (APPLY) {
    if (a.dbias == nullptr) return;
#pragma unroll
    for (int k = 0; k < 4; ++k) atomicAdd(&red[c + k], (double)a1[k]);
    __syncthreads();
    for (int i = tid; i < C; i += THREADS) atomicAdd(a.dbias + i, red[i]);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      atomicAdd(&red[0 * C + c + k], (double)a1[k]);
      atomicAdd(&red[1 * C + c + k], (double)a2[k]);
      atomicAdd(&red[2 * C + c + k], (double)a3[k]);
    }
    if (a.amax != nullptr) {
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) {
        mx_du = fmaxf(mx_du, __shfl_xor_sync(0xffffffffu, mx_du, off));
        mx_xh = fmaxf(mx_xh, __shfl_xor_sync(0xffffffffu, mx_xh, off));
      }
      if ((tid & 31) == 0) {
        atomic_max_pos(&redm[0], mx_du);
        atomic_max_pos(&redm[1], mx_xh);
      }
    }
    __syncthreads();
    for (int i = tid; i < C; i += THREADS) {
      atomicAdd(a.S1 + i, red[0 * C + i]);
      atomicAdd(a.S2 + i, red[1 * C + i]);
      atomicAdd(a.dalpha + i, red[2 * C + i]);
    }
    if (a.amax != nullptr && tid == 0) {
      atomic_max_pos(a.amax, redm[0]);
      atomic_max_pos(a.amax + 1, redm[1]);
    }
  }
}

template <typename YT, typename GT, int DF, bool APPLY, typename TC>
int launch_cfg(const BnStreamArgs& a, cudaStream_t st) {
  Geo g;
  g.TT = TC::TE / a.C;
  g.tps = (a.T + g.TT - 1) / g.TT;
  g.total = (long)a.N * g.tps;
  const size_t smem = (size_t)TC::NS * TC::TE * (sizeof(YT) + sizeof(GT)) +
                      TC::NS * sizeof(uint64_t) + (size_t)3 * a.C * sizeof(double) +
                      2 * sizeof(float);
  auto kern = bn_bwd_stream_kernel<YT, GT, DF, APPLY, TC>;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)(TC::NS * TC::TE * 8 + 64 + 3 * 1024 * 8 + 8));
    if (e != cudaSuccess) {
      pase_set_error("bn_stream: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr_done = true;
  }
  long grid = 2L * pase_num_sms();
  if (grid > g.total) grid = g.total;
  PASE_LAUNCH(kern, (unsigned)grid, THREADS, smem, st, a, g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    pase_set_error("bn_stream: launch failed: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return PASE_OK;
}

int tile_elems() {
  static int v = 0;
  if (v == 0) {
    const char* e = getenv("PASE_B200_BN_TILE");
    v = (e && atoi(e) == 2048) ? 2048 : 4096;
  }
  return v;
}

template <typename YT, typename GT, int DF, bool APPLY>
int launch(const BnStreamArgs& a, cudaStream_t st) {
  if (tile_elems() == 2048 && a.C <= 512) return launch_cfg<YT, GT, DF, APPLY, TileCfg<2048, 6>>(a, st);
  return launch_cfg<YT, GT, DF, APPLY, TileCfg<4096, 3>>(a, st);
}

bool stream_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PASE_B200_BN_STREAM");
    v = (e && atoi(e) == 0) ? 0 : 1;
  }
  return v == 1;
}

}  // namespace

bool pase_bn_stream_ok(const BnStreamArgs& a) {
  if (!stream_enabled()) return false;
  const int C = a.C;
  if (C < 32 || C > 1024 || (C & (C - 1)) != 0) return false;       // C/4 must divide 256
  if (a.a_bf16 && !a.y_bf16) return false;
  const size_t ysz = a.y_bf16 ? 2 : 4, gsz = a.a_bf16 ? 2 : 4;
  if ((reinterpret_cast<uintptr_t>(a.y) & 15u) || (reinterpret_cast<uintptr_t>(a.s.A) & 15u))
    return false;
  if ((a.y_ss * ysz) % 16 || (a.s.a_ss * gsz) % 16 || (a.s.a_rs * gsz) % 16 ||
      ((long)a.s.padL * a.s.a_rs * gsz) % 16)
    return false;
  if (a.s.P && ((reinterpret_cast<uintptr_t>(a.s.P) & 15u) || a.s.p_ss % 4 || a.s.p_rs % 4))
    return false;
  if (a.s.B && ((reinterpret_cast<uintptr_t>(a.s.B) & 15u) || a.s.b_ss % 4 || a.s.b_rs % 4))
    return false;
  return true;
}

int pase_bn_stream_reduce(const BnStreamArgs& a, cudaStream_t st) {
  if (a.y_bf16) {
    if (a.a_bf16) return launch<__nv_bfloat16, __nv_bfloat16, PASE_FMT_BF16, false>(a, st);
    return launch<__nv_bfloat16, float, PASE_FMT_BF16, false>(a, st);
  }
  return launch<float, float, PASE_FMT_F32, false>(a, st);
}

int pase_bn_stream_apply(const BnStreamArgs& a, cudaStream_t st) {
  if (a.dst_fmt == PASE_FMT_BF16) {
    if (a.a_bf16) return launch<__nv_bfloat16, __nv_bfloat16, PASE_FMT_BF16, true>(a, st);
    return launch<__nv_bfloat16, float, PASE_FMT_BF16, true>(a, st);
  }
  if (a.dst_fmt == PASE_FMT_F16X2) return launch<float, float, PASE_FMT_F16X2, true>(a, st);
  return launch<float, float, PASE_FMT_F32, true>(a, st);
}
