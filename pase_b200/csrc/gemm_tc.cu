// wgmma / TMA implicit-GEMM kernels for sm_90a.
//
//   pase_tc_gemm_nt : C[map(m), n] = alpha * sum_k A[m, k] * B[n, k] + bias[n]
//       A is addressed through a plain (non-overlapping) 2-D tensor [a_rows x R]:
//       element (m, k) lives at row m + k / R, column k % R, so the implicit im2col
//       matrix of a strided convolution (R = stride * Cin) needs no materialisation
//       and no overlapping TMA strides.  B is [N x K], K-major.
//   pase_tc_gemm_tn : C[i, j] += alpha * sum_r A[r, i] * B[r, j]   (weight gradients)
//       both operands MN-major in global memory; split over the reduction, the splits'
//       partial tiles summed in a fixed order (run-to-run identical results).  16-bit
//       operands are read MN-major by wgmma (transpose bits); tf32 wgmma only reads K-major
//       shared memory, so fp32 tiles are transposed in shared memory first.
//
// Numerics (`mode`), fp32 accumulation in registers in every mode:
//   0  TF32    .tf32 wgmma, fp32 operands read as tf32 (10-bit mantissa);
//   1  3xTF32  error-compensated: operands pre-split into exactly representable tf32 "hi"
//              and "lo" parts, D = Ahi*Bhi + Alo*Bhi + Ahi*Blo -> fp32-equivalent products;
//   2  BF16    .bf16 wgmma (one pass at twice the TF32 rate, half the bytes);
//   3  3xF16   error-compensated fp16: x = hi + 2^-11 lo', hi = rn_f16(x),
//              lo' = rn_f16((x - hi) 2^11) (both 11-bit significands -> 22-bit products like
//              3xTF32, at half the tensor time and half the operand bytes).  The scaled
//              correction products go to a SECOND register accumulator:
//              D = [Ahi*Bhi] + 2^-11 [Alo'*Bhi + Ahi*Blo'].  Operands must fit fp16's range
//              (gradients are pre-scaled by a power of two; `alpha_dev` undoes it).
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread issues), warpgroups 1 and 2
// = consumers; consumer warpgroup w issues the m64 wgmmas of tile rows [64 (w-1), +64) and runs
// their epilogue straight from the accumulator registers.  Operand tiles are 128-byte rows with
// the 128B swizzle.
#include "common.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdlib>

namespace {

constexpr int BM = 128;
constexpr uint32_t SPIN_LIMIT = 16u * 1000u * 1000u;   // >> any legitimate wait (each poll suspends)
constexpr float F16_LO_SCALE = 1.0f / 2048.0f;       // 2^-11, see pase_split_f16

// ---- numerics modes ------------------------------------------------------------------
template <int MODE>
struct ModeT {
  static constexpr int ESZ = MODE >= 2 ? 2 : 4;            // operand element size
  static constexpr bool SPLIT = (MODE == 1 || MODE == 3);  // hi/lo operands, 3 MMAs / product
  static constexpr int NACC = MODE == 3 ? 2 : 1;           // register accumulators
  static constexpr int EB = 128 / ESZ;                     // elements per 128-byte row
  static constexpr int KIND = MODE <= 1 ? 0 : (MODE == 2 ? 1 : 2);   // tf32 / bf16 / f16
};

// ------------------------------------------------------------------ PTX helpers ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// A wait that never completes is a pipeline bug or a bad tensor map: record (tag, block,
// thread) in a mapped host word (survives the trap; read back into pase_last_error()).
__device__ unsigned int* g_tc_diag = nullptr;
__device__ __noinline__ void mbar_timeout(int tag) {
  unsigned int* d = g_tc_diag;
  if (d != nullptr && atomicCAS(d, 0u, (unsigned)tag) == 0u) {
    d[1] = blockIdx.x + (blockIdx.y << 12) + (blockIdx.z << 24);
    d[2] = threadIdx.x;
    __threadfence_system();
  }
  __trap();
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > SPIN_LIMIT) mbar_timeout(tag);
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tmap_prefetch(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// the producer warpgroup hands registers to the two consumer warpgroups (40 + 2 x 232 per
// thread x 128 threads <= 64 K): the 3xF16 consumer holds three 64-register accumulators
__device__ __forceinline__ void regs_producer() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
}
__device__ __forceinline__ void regs_consumer() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
}
// the 256 consumer threads only
__device__ __forceinline__ void consumer_sync() {
  asm volatile("bar.sync 1, 256;" ::: "memory");
}
// this warp no longer reads the pipeline stage guarded by `bar` (8 arrivals free it)
__device__ __forceinline__ void release_stage(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

// ---- wgmma --------------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90 GMMA descriptor): start address, leading and stride
// byte offsets (all >> 4), layout type 1 = 128B swizzle at bits 62-63.
//   K-major : rows of 128 B, 8-row atoms of 1024 B -> SBO = 1024 B, LBO unused.
//   MN-major: 128 B (64 16-bit elements) along MN per k-row, 8 k-rows per 1024 B atom:
//             SBO = 1024 B (next 8 k), LBO = byte distance between 64-element MN blocks.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes,
                                              uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_wait0() {
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// keeps the compiler from touching accumulator registers across the asynchronous wgmma
template <int NR>
__device__ __forceinline__ void fence_regs(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int K>
struct KindTag {};

// accumulator register list / operand constraints, then the numbers of the operands after
// them (descriptors, scale-d, transpose immediates), per accumulator size
#define PASE_D32 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, " \
  "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define PASE_O32 \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), \
  "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), \
  "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), \
  "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), \
  "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define PASE_AB32 "%32, %33, p, 1, 1"
#define PASE_SC32 "%34"
#define PASE_TR32 ", %35, %36"
#define PASE_D64 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, " \
  "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, " \
  "%34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, " \
  "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define PASE_O64 \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), \
  "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), \
  "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), \
  "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), \
  "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), \
  "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), \
  "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), \
  "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
  "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), \
  "+f"(d[63])
#define PASE_AB64 "%64, %65, p, 1, 1"
#define PASE_SC64 "%66"
#define PASE_TR64 ", %67, %68"
// m64nNk{8,16} wgmma with fp32 accumulators d (N/2 registers per thread); scale_d = 0
// overwrites d.  TA / TB: operand MN-major (16-bit kinds only).
#define PASE_WGMMA(NR, KIND, INSTR, TRANS, ...)                                              \
  template <int TA, int TB>                                                                 \
  __device__ __forceinline__ void wgmma_call(float (&d)[NR], uint64_t da, uint64_t db,      \
                                             uint32_t scale_d, KindTag<KIND>) {             \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " PASE_SC##NR ", 0;\n\t" INSTR " "     \
                 PASE_D##NR ", " PASE_AB##NR TRANS ";\n\t}"                                   \
                 : PASE_O##NR                                                                \
                 : "l"(da), "l"(db), "r"(scale_d) __VA_ARGS__);                              \
  }
PASE_WGMMA(32, 0, "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32", "", )
PASE_WGMMA(32, 1, "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16", PASE_TR32, , "n"(TA), "n"(TB))
PASE_WGMMA(32, 2, "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16", PASE_TR32, , "n"(TA), "n"(TB))
PASE_WGMMA(64, 0, "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32", "", )
PASE_WGMMA(64, 1, "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16", PASE_TR64, , "n"(TA), "n"(TB))
PASE_WGMMA(64, 2, "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16", PASE_TR64, , "n"(TA), "n"(TB))
// The wgmmas of one 128-byte k-block: 4 k-steps of 32 B (+2 in the descriptor address when
// K-major, +kstep_desc in general).
//   plain : D += A*B;   3xTF32: D += Al*Bh + Ah*Bl + Ah*Bh (one accumulator);
//   3xF16 : Dc += Al'*Bh + Ah*Bl',  D += Ah*Bh.
template <int MODE, int TR, int NR, int NC>
__device__ __forceinline__ void issue_kblock(float (&acc)[NR], float (&corr)[NC], uint64_t dah,
                                             uint64_t dbh, uint64_t dal, uint64_t dbl,
                                             uint32_t kstep_desc, bool first) {
  using MT = ModeT<MODE>;
  constexpr KindTag<MT::KIND> kt{};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
    const uint64_t o = (uint64_t)(k * kstep_desc);
    if constexpr (MODE == 1) {
      wgmma_call<TR, TR>(acc, dal + o, dbh + o, sc, kt);
      wgmma_call<TR, TR>(acc, dah + o, dbl + o, 1u, kt);
      wgmma_call<TR, TR>(acc, dah + o, dbh + o, 1u, kt);
    } else if constexpr (MODE == 3) {
      wgmma_call<TR, TR>(corr, dal + o, dbh + o, sc, kt);
      wgmma_call<TR, TR>(corr, dah + o, dbl + o, 1u, kt);
      wgmma_call<TR, TR>(acc, dah + o, dbh + o, sc, kt);
    } else {
      wgmma_call<TR, TR>(acc, dah + o, dbh + o, sc, kt);
    }
  }
}

// Fold the finished accumulator(s) of one k-chunk into fp32 register sums with round-to-nearest
// adds: the split modes flush every K = 128, so rounding inside the tensor core's accumulation
// cannot drift over long reductions.
template <int MODE, int NR, int NC>
__device__ __forceinline__ void fold_chunk(float (&sums)[NR], const float (&acc)[NR],
                                           const float (&corr)[NC], bool first) {
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    float v = first ? acc[i] : sums[i] + acc[i];
    if constexpr (MODE == 3) v = fmaf(corr[i], F16_LO_SCALE, v);
    sums[i] = v;
  }
}

struct RowMap {
  int rows_in, t_valid, rows_out, fold, cols_per_fold;
};

constexpr int NTHREADS = 384;
constexpr int SMEM_LIMIT = 232448;                                    // 227 KB opt-in maximum
constexpr int BAR_BYTES = 256;
constexpr int MAX_STAGES = 8;

inline int pick_stages(int stage_bytes, int extra_bytes) {
  int st = (SMEM_LIMIT - 1024 - BAR_BYTES - extra_bytes) / stage_bytes;
  return st > MAX_STAGES ? MAX_STAGES : st;
}
inline int smem_bytes(int stages, int stage_bytes, int extra_bytes) {
  return stages * stage_bytes + 1024 + BAR_BYTES + extra_bytes;
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_f16(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}
// sum over the 8 lanes that share lane % 4 (the 8 accumulator rows g of a warp's m16 slice)
__device__ __forceinline__ float rowgroup_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

// Accumulator layout of m64nN (per warp: 16 rows): v[4j + 2h + e] = row g + 8h, column
// 8j + 2 t4 + e, with g = lane / 4, t4 = lane % 4.
struct Frag {
  int m[2];        // the two absolute rows of this thread
  int n0, t4, g;   // first column of the tile, lane % 4, lane / 4
};

struct NTArgs {
  int R;
  void* C;
  long ldc;
  int M, N, K;
  float alpha;
  const float* alpha_dev;          // optional device scalar multiplied into alpha
  const float* bias;
  RowMap rm;
  double* colsum;
  double* colsumsq;
  int accumulate, flush_kb, stages, stat_cols;
  // contextualised-MSE epilogue (fused regression head, tc_gemm_nt_kernel<.., CTX = true>):
  // C / cx_lo receive the fp16 pair of s * (prediction - label window) instead of the
  // prediction; cx_loss += sum d^2; cx_db[n] += sum_rows d
  const float* cx_label;           // (B, F, T) fp32
  int cx_F, cx_T, cx_r, cx_nvalid; // label geometry; columns >= cx_nvalid are padding (zeros)
  const float* cx_scale;           // device {1/s, s}
  void* cx_lo;
  double* cx_loss;
  double* cx_db;
};

// Output stage of the NT kernel: alpha / bias, row map and validity, store (fp32 or bf16),
// BatchNorm column statistics of the fp32 values (into shared-memory column sums).
template <int NR, bool OUT16>
__device__ __forceinline__ void nt_output(float (&v)[NR], const NTArgs& a, float alpha,
                                          const Frag& f, double* s_stats) {
  const int N = a.N;
  long orow[2];
  int nlim[2];                             // columns [0, nlim) of the row are valid
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = f.m[h];
    orow[h] = 0;
    nlim[h] = 0;
    if (m < a.M) {
      const int g = m / a.rm.rows_in;
      const int u = m - g * a.rm.rows_in;
      orow[h] = (long)g * a.rm.rows_out + u;
      const long lim = (long)(a.rm.t_valid - u * a.rm.fold) * a.rm.cols_per_fold;
      nlim[h] = lim <= 0 ? 0 : (lim >= N ? N : (int)lim);
    }
  }
  const bool want_stats = a.colsum != nullptr;
  const bool vec_ok = ((a.ldc & 1) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.C) & (OUT16 ? 3u : 7u)) == 0);
#pragma unroll
  for (int j = 0; j < NR / 4; ++j) {
    const int n = f.n0 + 8 * j + 2 * f.t4;
    const float b0 = (a.bias != nullptr && n < N) ? __ldg(a.bias + n) : 0.f;
    const float b1 = (a.bias != nullptr && n + 1 < N) ? __ldg(a.bias + n + 1) : 0.f;
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float x0 = fmaf(v[4 * j + 2 * h], alpha, b0);
      const float x1 = fmaf(v[4 * j + 2 * h + 1], alpha, b1);
      if constexpr (OUT16) {
        __nv_bfloat16* cp = reinterpret_cast<__nv_bfloat16*>(a.C) + orow[h] * a.ldc + n;
        if (n + 1 < nlim[h] && vec_ok) {
          *reinterpret_cast<uint32_t*>(cp) = pack_bf16(x0, x1);
        } else {
          if (n < nlim[h]) cp[0] = __float2bfloat16_rn(x0);
          if (n + 1 < nlim[h]) cp[1] = __float2bfloat16_rn(x1);
        }
      } else {
        float* cp = reinterpret_cast<float*>(a.C) + orow[h] * a.ldc + n;
        if (n + 1 < nlim[h] && vec_ok) {
          float2 o = make_float2(x0, x1);
          if (a.accumulate) {
            const float2 p = *reinterpret_cast<const float2*>(cp);
            o.x += p.x;
            o.y += p.y;
          }
          *reinterpret_cast<float2*>(cp) = o;
        } else {
          if (n < nlim[h]) cp[0] = a.accumulate ? cp[0] + x0 : x0;
          if (n + 1 < nlim[h]) cp[1] = a.accumulate ? cp[1] + x1 : x1;
        }
      }
      if (want_stats) {
        const float y0 = n < nlim[h] ? x0 : 0.f, y1 = n + 1 < nlim[h] ? x1 : 0.f;
        s1[0] += y0;
        s1[1] += y1;
        s2[0] = fmaf(y0, y0, s2[0]);
        s2[1] = fmaf(y1, y1, s2[1]);
      }
    }
    if (want_stats) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float c1 = rowgroup_sum(s1[e]), c2 = rowgroup_sum(s2[e]);
        if (f.g == 0 && n + e < N && (c1 != 0.f || c2 != 0.f)) {
          atomicAdd(&s_stats[n + e], (double)c1);
          atomicAdd(&s_stats[a.stat_cols + n + e], (double)c2);
        }
      }
    }
  }
}

// Output stage of the fused regression head (losses.py:15-37 + nn.MSELoss fused into the
// output GEMM of MLPMinion, minions.py:494-524): row m = (b, t); column n walks the
// (feature f, context slot j) pairs; label element = label[b][f][t + j - r/2] (zero outside).
template <int NR>
__device__ __forceinline__ void nt_output_ctx(const float (&v)[NR], const NTArgs& a, float alpha,
                                              const Frag& f, double& loss_acc) {
  const int NV = a.cx_nvalid, T = a.cx_T, F = a.cx_F, r = a.cx_r;
  const float s = __ldg(a.cx_scale + 1);
  int t[2];
  const float* lab[2];
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = f.m[h];
    row_ok[h] = m < a.M;
    const long b = row_ok[h] ? m / T : 0;
    t[h] = row_ok[h] ? (int)(m - b * T) : 0;
    lab[h] = a.cx_label + b * F * T;
  }
  float d2 = 0.f;
#pragma unroll
  for (int j = 0; j < NR / 4; ++j) {
    const int n = f.n0 + 8 * j + 2 * f.t4;      // n + 1 < a.N (= ldr, a multiple of 128)
    float cs[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float d[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int nn = n + e;
        float dd = 0.f;
        if (row_ok[h] && nn < NV) {
          const int ff = nn / r, jj = nn - ff * r;
          const float x = fmaf(v[4 * j + 2 * h + e], alpha, a.bias ? __ldg(a.bias + nn) : 0.f);
          const int tt = t[h] + jj - (r >> 1);
          const float lb = (tt >= 0 && tt < T) ? __ldg(lab[h] + (long)ff * T + tt) : 0.f;
          dd = x - lb;
        }
        d[e] = dd;
        cs[e] += dd;
        d2 = fmaf(dd, dd, d2);
      }
      if (row_ok[h]) {
        __half h0, l0, h1, l1;
        f16_split(d[0] * s, h0, l0);
        f16_split(d[1] * s, h1, l1);
        const long off = (long)f.m[h] * a.ldc + n;
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(a.C) + off) = pack_f16(h0, h1);
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(a.cx_lo) + off) = pack_f16(l0, l1);
      }
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {               // bias gradient: column sums of d
      const float c = rowgroup_sum(cs[e]);
      if (f.g == 0 && n + e < NV && c != 0.f) atomicAdd(a.cx_db + n + e, (double)c);
    }
  }
  loss_acc += (double)d2;
}

__device__ __forceinline__ void flush_stats(const NTArgs& a, const double* s_stats) {
  consumer_sync();
  for (int col = threadIdx.x - 128; col < a.N; col += 256) {
    const double s = s_stats[col], b2 = s_stats[a.stat_cols + col];
    if (s != 0.0 || b2 != 0.0) {
      atomicAdd(a.colsum + col, s);
      atomicAdd(a.colsumsq + col, b2);
    }
  }
}

// ------------------------------------------------------------------ NT kernel ----
// Persistent: CTA b processes tiles b, b+grid, ... (n-tile fastest so concurrently running
// CTAs share A rows in L2).  Stage = [A.hi | B.hi | A.lo | B.lo], each 128-byte K-major rows.
// The split modes accumulate `flush_kb` k-blocks in the wgmma accumulators, then fold them into
// fp32 register sums with round-to-nearest adds.
template <int BN, int MODE>
struct NTCfg {
  using MT = ModeT<MODE>;
  static constexpr int BK = 128 / MT::ESZ;                 // elements per k-block
  static constexpr int A_BYTES = BM * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = (MT::SPLIT ? 2 : 1) * (A_BYTES + B_BYTES);
  static constexpr int NR = BN / 2;                        // accumulator registers per thread
};

template <int BN, int MODE, bool OUT16, bool CTX>
__global__ void __launch_bounds__(NTHREADS, 1)
tc_gemm_nt_kernel(const __grid_constant__ CUtensorMap mAhi, const __grid_constant__ CUtensorMap mAlo,
                  const __grid_constant__ CUtensorMap mBhi, const __grid_constant__ CUtensorMap mBlo,
                  const NTArgs a) {
  using Cfg = NTCfg<BN, MODE>;
  using MT = ModeT<MODE>;
  constexpr int BK = Cfg::BK, NR = Cfg::NR;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int stages = a.stages;
  uint8_t* tiles = smem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + stages * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  // column sums in fp64: the order of the warps' additions then only moves bits that the
  // fp32 consumers of the statistics never see (run-to-run identical results)
  double* s_stats = reinterpret_cast<double*>(smem + stages * Cfg::STAGE_BYTES + BAR_BYTES);

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int M = a.M, N = a.N, K = a.K, R = a.R;
  const int n_tiles = (N + BN - 1) / BN, m_tiles = (M + BM - 1) / BM;
  const int total_tiles = n_tiles * m_tiles;
  const int nkb = (K + BK - 1) / BK;
  int flush_kb = a.flush_kb;
  if (flush_kb <= 0 || flush_kb > nkb) flush_kb = nkb;
  const int nchunks = (nkb + flush_kb - 1) / flush_kb;
  const bool want_stats = a.colsum != nullptr;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);                     // one arrival per consumer warp
    }
    fence_barrier_init();
    tmap_prefetch(&mAhi);
    tmap_prefetch(&mBhi);
    if (MT::SPLIT) {
      tmap_prefetch(&mAlo);
      tmap_prefetch(&mBlo);
    }
  }
  if (want_stats)
    for (int i = threadIdx.x; i < 2 * a.stat_cols; i += NTHREADS) s_stats[i] = 0.0;
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    regs_producer();
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
        int arow = m0, acol = 0;                 // folded-row view: k = (arow - m0) * R + acol
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty_bar[s], ph ^ 1, 1);
          uint8_t* st = tiles + s * Cfg::STAGE_BYTES;
          mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
          const int kf = kb * BK;
          tma_load_2d(st, &mAhi, &full_bar[s], acol, arow);
          tma_load_2d(st + Cfg::A_BYTES, &mBhi, &full_bar[s], kf, n0);
          if (MT::SPLIT) {
            tma_load_2d(st + Cfg::A_BYTES + Cfg::B_BYTES, &mAlo, &full_bar[s], acol, arow);
            tma_load_2d(st + 2 * Cfg::A_BYTES + Cfg::B_BYTES, &mBlo, &full_bar[s], kf, n0);
          }
          acol += BK;
          while (acol >= R) {
            acol -= R;
            ++arow;
          }
          if (++s == stages) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
    return;
  }

  regs_consumer();
  const int cw = wg - 1;                          // rows [64 cw, +64) of every tile
  const int wq = (threadIdx.x >> 5) & 3;
  Frag f;
  f.g = lane >> 2;
  f.t4 = lane & 3;
  const float alpha = a.alpha * (a.alpha_dev ? __ldg(a.alpha_dev) : 1.f);
  const uint32_t tiles_u32 = smem_u32(tiles);
  const uint64_t dconst = make_desc(0, 16, 1024);
  float acc[NR];
  float corr[MT::NACC == 2 ? NR : 1];
  float sums[MT::SPLIT ? NR : 1];
  double cx_loss = 0.0;
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
    for (int ch = 0; ch < nchunks; ++ch) {
      const int kb_lo = ch * flush_kb;
      const int kb_hi = (kb_lo + flush_kb < nkb) ? kb_lo + flush_kb : nkb;
      for (int kb = kb_lo; kb < kb_hi; ++kb) {
        mbar_wait(&full_bar[s], ph, 2);
        const uint32_t st = tiles_u32 + s * Cfg::STAGE_BYTES;
        const uint64_t dah = dconst + ((st + cw * 64 * 128) >> 4);
        const uint64_t dbh = dconst + ((st + Cfg::A_BYTES) >> 4);
        const uint64_t dal = dconst + ((st + Cfg::A_BYTES + Cfg::B_BYTES + cw * 64 * 128) >> 4);
        const uint64_t dbl = dconst + ((st + 2 * Cfg::A_BYTES + Cfg::B_BYTES) >> 4);
        wgmma_fence();
        issue_kblock<MODE, 0>(acc, corr, dah, dbh, dal, dbl, 2, kb == kb_lo);
        wgmma_commit();
        // drained per k-block: with 3 stages of 64 KB (3xF16), holding a stage for one more
        // k-block (wait_group 1) starves the producer; it measured 5 % slower on an H100
        wgmma_wait0();
        fence_regs(acc);
        fence_regs(corr);
        release_stage(&empty_bar[s], lane);
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
      if constexpr (MT::SPLIT) fold_chunk<MODE>(sums, acc, corr, ch == 0);
    }
    f.m[0] = m0 + cw * 64 + wq * 16 + f.g;
    f.m[1] = f.m[0] + 8;
    f.n0 = n0;
    if constexpr (CTX) {
      if constexpr (MT::SPLIT) nt_output_ctx<NR>(sums, a, alpha, f, cx_loss);
      else nt_output_ctx<NR>(acc, a, alpha, f, cx_loss);
    } else {
      if constexpr (MT::SPLIT) nt_output<NR, OUT16>(sums, a, alpha, f, s_stats);
      else nt_output<NR, OUT16>(acc, a, alpha, f, s_stats);
    }
  }
  if constexpr (CTX) {
    cx_loss = warp_sum_d(cx_loss);
    if (lane == 0 && cx_loss != 0.0) atomicAdd(a.cx_loss, cx_loss);
  }
  if (want_stats) flush_stats(a, s_stats);
}

// ------------------------------------------------------------------ TN kernel ----
// C[i,j] += alpha * sum_r A[r,i] B[r,j].  A: 4-D tensor (128 B inner, rows-per-group, column
// blocks, groups); B addressed through the folded-row trick: (r, j) -> row u + j/R of group g,
// column j % R.  One stage = KR reduction rows (4 wgmma k-steps): 32 rows of fp32, 64 of 16-bit,
// stored as MN blocks of [KR rows x 128 B].
//   16-bit: wgmma reads the MN-major blocks directly (128B swizzle, LBO = next MN block).
//   fp32  : the consumers transpose each stage into K-major 128B-swizzled tiles [MN x 128 B]
//           (tf32 wgmma has no MN-major form) and run the NT k-block on them.
template <int BN, int MODE>
struct TNCfg {
  using MT = ModeT<MODE>;
  static constexpr int EB = MT::EB;                        // elements per 128-byte MN block
  static constexpr int KR = 4 * 32 / MT::ESZ;              // reduction rows per stage
  static constexpr int A_BYTES = KR * BM * MT::ESZ;        // BM/EB MN-blocks of [KR rows x 128 B]
  static constexpr int B_BYTES = KR * BN * MT::ESZ;
  static constexpr int STAGE_BYTES = (MT::SPLIT ? 2 : 1) * (A_BYTES + B_BYTES);
  static constexpr bool TRANSPOSE = MT::ESZ == 4;
  static constexpr int T_BYTES = TRANSPOSE ? STAGE_BYTES : 0;   // K-major copy of one stage
  static constexpr int LBO = KR * 128;                     // next MN block
  static constexpr int NR = BN / 2;
};

struct TNArgs {
  int R;
  float* C;
  long ldc;
  int I, J, groups, rows_per_group;
  float alpha;
  const float* alpha_dev;
  int chunks_per_split, flush_ch, stages, b_blocked, accumulate;
  float* ws;                       // several splits: [split][tile][BM x BN] partial tiles
};

// fp32 stage operand [rows/32 blocks of (32 k-rows x 32 elements)] -> K-major 128B-swizzled
// [rows x 32 k] (row i, k at byte i*128 + ((k/4 ^ i%8) * 16) + (k%4) * 4)
template <int ROWS>
__device__ __forceinline__ void transpose_tile(const float* __restrict__ src, float* __restrict__ dst,
                                               int ctid) {
#pragma unroll 4
  for (int e = ctid; e < 32 * ROWS; e += 256) {
    const int k = e / ROWS, i = e % ROWS;
    dst[i * 32 + ((((k >> 2) ^ (i & 7))) << 2) + (k & 3)] = src[(i >> 5) * 1024 + k * 32 + (i & 31)];
  }
}

// alpha * (this warp's 16 tile rows starting at r0).  One split: straight into C (C = x, or
// C += x when accumulating; every element has exactly one writer).  Several splits: into this
// split's partial tile in the workspace, which tn_reduce_splits_kernel sums in split order, so
// the result does not depend on the order in which the splits finish.
template <int BN, int NR>
__device__ __forceinline__ void tn_output(const float (&v)[NR], const TNArgs& a, int r0, int i0,
                                          int j0, int lane) {
  const float alpha = a.alpha * (a.alpha_dev ? __ldg(a.alpha_dev) : 1.f);
  const bool vec_ok = ((a.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(a.C) & 7u) == 0);
  const int g = lane >> 2, t4 = lane & 3;
  float* tile = a.ws == nullptr ? nullptr
      : a.ws + (((long)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * (BM * BN);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + g + 8 * h, i = i0 + r;
    if (tile == nullptr && i >= a.I) continue;
    float* crow = a.C + (long)i * a.ldc;
#pragma unroll
    for (int j = 0; j < NR / 4; ++j) {
      const int col = 8 * j + 2 * t4, n = j0 + col;
      const float x0 = v[4 * j + 2 * h] * alpha, x1 = v[4 * j + 2 * h + 1] * alpha;
      if (tile != nullptr) {
        *reinterpret_cast<float2*>(tile + r * BN + col) = make_float2(x0, x1);
      } else if (n + 1 < a.J && vec_ok) {
        float2 o = make_float2(x0, x1);
        if (a.accumulate) {
          const float2 p = *reinterpret_cast<const float2*>(crow + n);
          o.x += p.x;
          o.y += p.y;
        }
        *reinterpret_cast<float2*>(crow + n) = o;
      } else {
        if (n < a.J) crow[n] = a.accumulate ? crow[n] + x0 : x0;
        if (n + 1 < a.J) crow[n + 1] = a.accumulate ? crow[n + 1] + x1 : x1;
      }
    }
  }
}

// C[i, j] (+)= sum over the splits, in split order, of the partial tiles holding (i, j)
__global__ void tn_reduce_splits_kernel(const float* __restrict__ ws, int splits, int tiles_j,
                                        int bn, long tiles, float* __restrict__ C, long ldc, int I,
                                        int J, int accumulate) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)I * J) return;
  const int i = (int)(idx / J), j = (int)(idx % J);
  const long tile_elems = (long)BM * bn;
  const float* p = ws + ((long)(i / BM) * tiles_j + j / bn) * tile_elems + (i % BM) * bn + j % bn;
  float sum = 0.f;
  for (int z = 0; z < splits; ++z) sum += p[z * tiles * tile_elems];
  float* c = C + (long)i * ldc + j;
  *c = accumulate ? *c + sum : sum;
}

template <int BN, int MODE>
__global__ void __launch_bounds__(NTHREADS, 1)
tc_gemm_tn_kernel(const __grid_constant__ CUtensorMap mAhi, const __grid_constant__ CUtensorMap mAlo,
                  const __grid_constant__ CUtensorMap mBhi, const __grid_constant__ CUtensorMap mBlo,
                  const TNArgs a) {
  using Cfg = TNCfg<BN, MODE>;
  using MT = ModeT<MODE>;
  constexpr int KR = Cfg::KR, EB = Cfg::EB, NR = Cfg::NR;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int stages = a.stages;
  uint8_t* tiles = smem;
  uint8_t* ttile = smem + stages * Cfg::STAGE_BYTES;                 // transposed stage (fp32)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ttile + Cfg::T_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int R = a.R;
  const int j0 = blockIdx.x * BN, i0 = blockIdx.y * BM;
  const int cpg = (a.rows_per_group + KR - 1) / KR;           // chunks per group
  const long total_chunks = (long)a.groups * cpg;
  const long c_begin = (long)blockIdx.z * a.chunks_per_split;
  long c_end = c_begin + a.chunks_per_split;
  if (c_end > total_chunks) c_end = total_chunks;
  const int nch = (int)(c_end - c_begin);
  if (nch <= 0) return;                // uniform across the CTA
  int flush_ch = a.flush_ch;
  if (flush_ch <= 0 || flush_ch > nch) flush_ch = nch;
  const int nflush = (nch + flush_ch - 1) / flush_ch;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    fence_barrier_init();
    tmap_prefetch(&mAhi);
    tmap_prefetch(&mBhi);
  }
  __syncthreads();
  pdl_wait();
  const int jq = j0 / R, jc = j0 % R;  // folded-row offset / column of this B tile

  if (wg == 0) {
    regs_producer();
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int it = 0; it < nch; ++it) {
        mbar_wait(&empty_bar[s], ph ^ 1, 11);
        const long ch = c_begin + it;
        const int g = (int)(ch / cpg);
        const int u0 = (int)(ch - (long)g * cpg) * KR;
        uint8_t* st = tiles + s * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
        uint8_t* a_hi = st;
        uint8_t* b_hi = st + Cfg::A_BYTES;
        uint8_t* a_lo = b_hi + Cfg::B_BYTES;
        uint8_t* b_lo = a_lo + Cfg::A_BYTES;
        // A: one 4-D box = (128 B, KR rows, BM/EB column blocks, 1 group) lands as
        // BM/EB consecutive [KR rows x 128 B] MN-blocks
        tma_load_4d(a_hi, &mAhi, &full_bar[s], 0, u0, i0 / EB, g);
        if (MT::SPLIT) tma_load_4d(a_lo, &mAlo, &full_bar[s], 0, u0, i0 / EB, g);
        if (a.b_blocked) {
          // the BN columns of this tile lie inside one folded row (R % BN == 0)
          tma_load_4d(b_hi, &mBhi, &full_bar[s], 0, u0 + jq, jc / EB, g);
          if (MT::SPLIT) tma_load_4d(b_lo, &mBlo, &full_bar[s], 0, u0 + jq, jc / EB, g);
        } else {
#pragma unroll
          for (int nb = 0; nb < BN / EB; ++nb) {
            // EB consecutive columns never straddle a folded row (R % EB == 0)
            const int col = jc + nb * EB;
            const int qq = jq + col / R, cc = col % R;
            tma_load_4d(b_hi + nb * KR * 128, &mBhi, &full_bar[s], 0, u0 + qq, cc / EB, g);
            if (MT::SPLIT)
              tma_load_4d(b_lo + nb * KR * 128, &mBlo, &full_bar[s], 0, u0 + qq, cc / EB, g);
          }
        }
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  regs_consumer();
  const int cw = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3;
  const int ctid = threadIdx.x - 128;
  // K-major (transposed fp32) or MN-major (16-bit) descriptors; WG cw's 64 A rows start
  // 64 * 128 B into the K-major tile, one MN block (KR * 128 B) into the MN-major stage
  const uint64_t dconst = Cfg::TRANSPOSE ? make_desc(0, 16, 1024) : make_desc(0, Cfg::LBO, 1024);
  const uint32_t kstep = Cfg::TRANSPOSE ? 2u : (uint32_t)((16 * 128) >> 4);
  float acc[NR];
  float corr[MT::NACC == 2 ? NR : 1];
  float sums[MT::SPLIT ? NR : 1];
  int s = 0;
  uint32_t ph = 0;
  for (int fl = 0; fl < nflush; ++fl) {
    const int it_lo = fl * flush_ch;
    const int it_hi = (it_lo + flush_ch < nch) ? it_lo + flush_ch : nch;
    for (int it = it_lo; it < it_hi; ++it) {
      mbar_wait(&full_bar[s], ph, 12);
      uint32_t base;
      if constexpr (Cfg::TRANSPOSE) {
        consumer_sync();               // both warpgroups' previous wgmmas have retired
        const float* st = reinterpret_cast<const float*>(tiles + s * Cfg::STAGE_BYTES);
        float* tt = reinterpret_cast<float*>(ttile);
        transpose_tile<BM>(st, tt, ctid);
        transpose_tile<BN>(st + Cfg::A_BYTES / 4, tt + Cfg::A_BYTES / 4, ctid);
        if constexpr (MT::SPLIT) {
          const int o = (Cfg::A_BYTES + Cfg::B_BYTES) / 4;
          transpose_tile<BM>(st + o, tt + o, ctid);
          transpose_tile<BN>(st + o + Cfg::A_BYTES / 4, tt + o + Cfg::A_BYTES / 4, ctid);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        consumer_sync();
        release_stage(&empty_bar[s], lane);
        base = smem_u32(ttile);
      } else {
        base = smem_u32(tiles + s * Cfg::STAGE_BYTES);
      }
      const uint32_t a_off = Cfg::TRANSPOSE ? cw * 64 * 128 : cw * Cfg::LBO;
      const uint64_t dah = dconst + ((base + a_off) >> 4);
      const uint64_t dbh = dconst + ((base + Cfg::A_BYTES) >> 4);
      const uint64_t dal = dconst + ((base + Cfg::A_BYTES + Cfg::B_BYTES + a_off) >> 4);
      const uint64_t dbl = dconst + ((base + 2 * Cfg::A_BYTES + Cfg::B_BYTES) >> 4);
      wgmma_fence();
      issue_kblock<MODE, Cfg::TRANSPOSE ? 0 : 1>(acc, corr, dah, dbh, dal, dbl, kstep, it == it_lo);
      wgmma_commit();
      wgmma_wait0();
      fence_regs(acc);
      fence_regs(corr);
      if constexpr (!Cfg::TRANSPOSE) release_stage(&empty_bar[s], lane);
      if (++s == stages) {
        s = 0;
        ph ^= 1;
      }
    }
    if constexpr (MT::SPLIT) fold_chunk<MODE>(sums, acc, corr, fl == 0);
  }
  if constexpr (MT::SPLIT) tn_output<BN, NR>(sums, a, cw * 64 + wq * 16, i0, j0, lane);
  else tn_output<BN, NR>(acc, a, cw * 64 + wq * 16, i0, j0, lane);
}

// ------------------------------------------------------------------ host side ----
// A timed-out mbarrier wait traps the kernel; the (tag, block, thread) it recorded in the
// mapped host diagnostics word is appended to the error message of the failing call.
static unsigned int* h_tc_diag = nullptr;
static void pase_tc_init_diag() {
  static bool done = false;
  if (done) return;
  done = true;
  unsigned int* h = nullptr;
  unsigned int* d = nullptr;
  // 16 bytes of mapped pinned memory, allocated once per process (diagnostics only)
  if (cudaHostAlloc((void**)&h, 4 * sizeof(unsigned int), cudaHostAllocMapped) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  h[0] = h[1] = h[2] = h[3] = 0;
  if (cudaHostGetDevicePointer((void**)&d, h, 0) != cudaSuccess ||
      cudaMemcpyToSymbol(g_tc_diag, &d, sizeof(d)) != cudaSuccess) {
    cudaGetLastError();
    cudaFreeHost(h);
    return;
  }
  h_tc_diag = h;
}
static void pase_tc_report_timeout() {
  if (h_tc_diag != nullptr && h_tc_diag[0] != 0)
    pase_set_error("pase tc gemm: mbarrier wait timed out (tag %u, block code 0x%x, thread %u)",
                   h_tc_diag[0], h_tc_diag[1], h_tc_diag[2]);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || p == nullptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// rank-2 .. rank-4 tensor map (element type by mode), zero OOB fill.
int make_map(CUtensorMap* map, const void* base, int mode, int rank, const uint64_t* dims,
             const uint64_t* strides_bytes, const uint32_t* box, const char* what,
             CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    pase_set_error("pase tc gemm: cuTensorMapEncodeTiled not available");
    return PASE_ERR_UNSUPPORTED;
  }
  const CUtensorMapDataType dt = mode <= 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                           : (mode == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                        : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base),
                   (const cuuint64_t*)dims, (const cuuint64_t*)strides_bytes,
                   (const cuuint32_t*)box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    pase_set_error("pase tc gemm: cuTensorMapEncodeTiled(%s) failed with %d (dims %llu,%llu,%llu "
                   "stride %llu,%llu box %u,%u,%u)",
                   what, (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1],
                   (unsigned long long)(rank > 2 ? dims[2] : 0),
                   (unsigned long long)strides_bytes[0],
                   (unsigned long long)(rank > 2 ? strides_bytes[1] : 0), box[0], box[1],
                   rank > 2 ? box[2] : 0);
    return PASE_ERR_ARG;
  }
  return PASE_OK;
}

#define PASE_TC_LAUNCH_CHECK(name)                                         \
  do {                                                                     \
    cudaError_t e__ = cudaGetLastError();                                  \
    if (e__ != cudaSuccess) {                                              \
      pase_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      pase_tc_report_timeout();                                            \
      return (int)e__;                                                     \
    }                                                                      \
  } while (0)

template <int BN, int MODE, bool OUT16, bool CTX>
int launch_nt(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh,
              const CUtensorMap& bl, NTArgs a, cudaStream_t st) {
  using Cfg = NTCfg<BN, MODE>;
  static bool attr = false;
  a.stat_cols = a.colsum ? ((a.N + 31) / 32) * 32 : 0;
  a.stages = pick_stages(Cfg::STAGE_BYTES, 2 * a.stat_cols * 8);
  const int smem = smem_bytes(a.stages, Cfg::STAGE_BYTES, 2 * a.stat_cols * 8);
  if (a.stages < 2) {
    pase_set_error("pase_tc_gemm_nt: not enough shared memory for 2 pipeline stages");
    return PASE_ERR_UNSUPPORTED;
  }
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tc_gemm_nt_kernel<BN, MODE, OUT16, CTX>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) {
      pase_set_error("pase_tc_gemm_nt: smem attribute: %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr = true;
  }
  const long tiles = (long)((a.N + BN - 1) / BN) * ((a.M + BM - 1) / BM);
  const int grid = (int)(tiles < pase_num_sms() ? tiles : pase_num_sms());
  PASE_LAUNCH((tc_gemm_nt_kernel<BN, MODE, OUT16, CTX>), grid, NTHREADS, smem, st, ah, al, bh, bl, a);
  PASE_TC_LAUNCH_CHECK(CTX ? "pase_tc_gemm_nt_ctxmse" : "pase_tc_gemm_nt");
  return PASE_OK;
}

// Partial tiles of the split weight-gradient GEMM: room for 4 CTAs per SM of BM x 128 fp32,
// allocated once per device on first use (never freed: captured CUDA graphs keep using it).
static float* tn_workspace(cudaStream_t st) {
  static float* ws[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) {
    pase_set_error("pase_tc_gemm_tn: device index %d", dev);
    return nullptr;
  }
  if (ws[dev] != nullptr) return ws[dev];
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  if (cs != cudaStreamCaptureStatusNone) {
    pase_set_error("pase_tc_gemm_tn: first split-K call on this device inside a stream capture "
                   "(run one step before capturing)");
    return nullptr;
  }
  cudaError_t e = cudaMalloc(&ws[dev], (size_t)4 * pase_num_sms() * BM * 128 * sizeof(float));
  if (e != cudaSuccess) {
    ws[dev] = nullptr;
    pase_set_error("pase_tc_gemm_tn: workspace allocation: %s", cudaGetErrorString(e));
    return nullptr;
  }
  return ws[dev];
}

template <int BN, int MODE>
int launch_tn(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh,
              const CUtensorMap& bl, TNArgs a, cudaStream_t st) {
  using Cfg = TNCfg<BN, MODE>;
  static bool attr = false;
  a.stages = pick_stages(Cfg::STAGE_BYTES, Cfg::T_BYTES);
  const int smem = smem_bytes(a.stages, Cfg::STAGE_BYTES, Cfg::T_BYTES);
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tc_gemm_tn_kernel<BN, MODE>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) {
      pase_set_error("pase_tc_gemm_tn: smem attribute: %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr = true;
  }
  const int ti = (a.I + BM - 1) / BM, tj = (a.J + BN - 1) / BN;
  const int cpg = (a.rows_per_group + Cfg::KR - 1) / Cfg::KR;
  const long total = (long)a.groups * cpg;
  // split the reduction so that the CTA count fills whole waves of the SMs (one CTA per SM):
  // among 1..4 waves pick the split with the best fill, keeping chains >= 8 chunks
  const long tiles = (long)ti * tj;
  const int sms = pase_num_sms();
  long best = 1;
  double best_eff = -1.0;
  for (long sp = 1; sp <= total && sp * tiles <= 4L * sms; ++sp) {
    const long cps_try = (total + sp - 1) / sp;
    if (cps_try < 8 && sp > 1) break;
    const long ctas = tiles * ((total + cps_try - 1) / cps_try);
    const long waves = (ctas + sms - 1) / sms;
    // time ~ waves * chunks-per-cta: lower is better
    const double cost = (double)waves * (double)(cps_try + 6);
    const double eff = 1.0 / cost;
    if (eff > best_eff) { best_eff = eff; best = sp; }
  }
  long splits = best;
  long cps = (total + splits - 1) / splits;
  splits = (total + cps - 1) / cps;
  a.chunks_per_split = (int)cps;
  a.ws = nullptr;
  if (splits > 1) {      // splits * tiles <= 4 * sms CTAs (loop above): fits the workspace
    if ((a.ws = tn_workspace(st)) == nullptr) return PASE_ERR_UNSUPPORTED;
  }
  dim3 grid(tj, ti, (unsigned)splits);
  PASE_LAUNCH((tc_gemm_tn_kernel<BN, MODE>), grid, NTHREADS, smem, st, ah, al, bh, bl, a);
  PASE_TC_LAUNCH_CHECK("pase_tc_gemm_tn");
  if (splits > 1) {
    const long n = (long)a.I * a.J;
    tn_reduce_splits_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        a.ws, (int)splits, tj, BN, tiles, a.C, a.ldc, a.I, a.J, a.accumulate);
    PASE_TC_LAUNCH_CHECK("pase_tc_gemm_tn (split reduction)");
  }
  return PASE_OK;
}

// tf32 helpers: the tensor core reads the upper 19 bits of an fp32 operand (truncation).
__device__ __forceinline__ float tf32_trunc(float v) {
  return __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
}
__device__ __forceinline__ float tf32_rn(float v) {          // round to nearest even
  uint32_t u = __float_as_uint(v);
  u += 0xFFFu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xFFFFE000u);
}
// split kernel.
//   hi == nullptr (activations): the operand itself is "hi" (hardware truncation), and
//        lo = rn(x - trunc(x));
//   hi != nullptr (weights): hi = rn(x), lo = rn(x - hi): explicit, exactly representable,
//        zero-mean residuals, so the dropped lo*lo / residual terms carry no coherent bias.
__global__ void split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi,
                                  float* __restrict__ lo, long n) {
  const long i4 = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const long stride = (long)gridDim.x * blockDim.x * 4;
  const bool explicit_hi = hi != nullptr;
  for (long i = i4; i < n; i += stride) {
    if (i + 3 < n) {
      const float4 v = *reinterpret_cast<const float4*>(x + i);
      const float vv[4] = {v.x, v.y, v.z, v.w};
      float h[4], l[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        h[k] = explicit_hi ? tf32_rn(vv[k]) : tf32_trunc(vv[k]);
        l[k] = tf32_rn(vv[k] - h[k]);
      }
      if (explicit_hi) *reinterpret_cast<float4*>(hi + i) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(lo + i) = make_float4(l[0], l[1], l[2], l[3]);
    } else {
      for (long j = i; j < n; ++j) {
        const float v = x[j];
        const float h = explicit_hi ? tf32_rn(v) : tf32_trunc(v);
        if (explicit_hi) hi[j] = h;
        lo[j] = tf32_rn(v - h);
      }
    }
  }
}

}  // namespace

extern "C" {

int pase_split_tf32(const float* x, float* hi, float* lo, long n, void* stream) {
  // hi may be NULL: tf32 wgmma ignores the low 13 mantissa bits of its fp32 operands, so the
  // original array serves as "hi".
  PASE_CHECK_ARG(x && lo && n > 0, "pase_split_tf32: bad args");
  PASE_CHECK_ARG(aligned16(x) && aligned16(lo) && (hi == nullptr || aligned16(hi)),
                 "pase_split_tf32: alignment");
  long blocks = (n / 4 + 255) / 256;
  long cap = (long)pase_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  split_tf32_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, hi, lo, n);
  PASE_LAUNCH_CHECK("pase_split_tf32");
  return PASE_OK;
}

// A: [a_rows x R] elements (hi / lo parts; lo NULL outside the split modes); B: [N x K]
// (ldb >= K).  Element type by mode: fp32 (0, 1), bf16 (2), fp16 (3).
int pase_tc_gemm_nt(const void* Ahi, const void* Alo, long a_rows, int R, const void* Bhi,
                    const void* Blo, long ldb, void* C, long ldc, int M, int N, int K,
                    float alpha, const float* alpha_dev, const float* bias, int rows_in,
                    int t_valid, int rows_out, int fold, double* colsum, double* colsumsq,
                    int accumulate, int mode, int c_bf16, void* stream) {
  PASE_CHECK_ARG(Ahi && Bhi && C && M > 0 && N > 0 && K > 0, "pase_tc_gemm_nt: bad args");
  PASE_CHECK_ARG(mode >= 0 && mode <= 3, "pase_tc_gemm_nt: mode %d (0 tf32, 1 3xtf32, 2 bf16, "
                 "3 3xf16)", mode);
  pase_tc_init_diag();
  const bool split = mode == 1 || mode == 3;
  const int esz = mode >= 2 ? 2 : 4;
  const int eb = 128 / esz;                       // elements per 128-byte row
  PASE_CHECK_ARG(!split || (Alo && Blo), "pase_tc_gemm_nt: split modes need lo operands");
  PASE_CHECK_ARG(R >= eb && (R % eb) == 0, "pase_tc_gemm_nt: R=%d must be a multiple of %d", R,
                 eb);
  PASE_CHECK_ARG((K * esz) % 16 == 0 && (ldb * esz) % 16 == 0 && ldb >= K,
                 "pase_tc_gemm_nt: K/ldb alignment");
  PASE_CHECK_ARG(aligned16(Ahi) && aligned16(Bhi), "pase_tc_gemm_nt: operand alignment");
  PASE_CHECK_ARG(rows_in > 0 && rows_out > 0 && fold > 0 && (N % fold) == 0,
                 "pase_tc_gemm_nt: bad row map");
  PASE_CHECK_ARG((colsum == nullptr) == (colsumsq == nullptr), "pase_tc_gemm_nt: stats pair");
  PASE_CHECK_ARG(colsum == nullptr || N <= 4096, "pase_tc_gemm_nt: stats need N <= 4096");
  PASE_CHECK_ARG(colsum == nullptr || !accumulate, "pase_tc_gemm_nt: stats + accumulate");
  PASE_CHECK_ARG(!c_bf16 || !accumulate, "pase_tc_gemm_nt: bf16 output cannot accumulate");
  const int BN = N <= 64 ? 64 : 128;
  const int bk = eb;
  // split modes: fold the accumulators into fp32 register sums every K = 128; over K <= 512
  // the tensor core's own accumulation stays below 1e-6 relative, so short reductions (sinc
  // layer, block-1 dgrad) keep one chunk
  const int flush_kb = (split && K > 512) ? 128 / bk : 0;
  CUtensorMap ah, al, bh, bl;
  uint64_t adims[2] = {(uint64_t)R, (uint64_t)a_rows};
  uint64_t astr[1] = {(uint64_t)R * esz};
  uint32_t abox[2] = {(uint32_t)bk, (uint32_t)BM};
  uint64_t bdims[2] = {(uint64_t)K, (uint64_t)N};
  uint64_t bstr[1] = {(uint64_t)ldb * esz};
  uint32_t bbox[2] = {(uint32_t)bk, (uint32_t)BN};
  int rc;
  if ((rc = make_map(&ah, Ahi, mode, 2, adims, astr, abox, "A.hi")) != 0) return rc;
  if ((rc = make_map(&bh, Bhi, mode, 2, bdims, bstr, bbox, "B.hi")) != 0) return rc;
  if (split) {
    if ((rc = make_map(&al, Alo, mode, 2, adims, astr, abox, "A.lo")) != 0) return rc;
    if ((rc = make_map(&bl, Blo, mode, 2, bdims, bstr, bbox, "B.lo")) != 0) return rc;
  } else {
    al = ah;
    bl = bh;
  }
  NTArgs a;
  a.R = R; a.C = C; a.ldc = ldc; a.M = M; a.N = N; a.K = K; a.alpha = alpha;
  a.alpha_dev = alpha_dev; a.bias = bias;
  a.rm = RowMap{rows_in, t_valid, rows_out, fold, N / fold};
  a.colsum = colsum; a.colsumsq = colsumsq; a.accumulate = accumulate; a.flush_kb = flush_kb;
  a.stages = 0; a.stat_cols = 0;
  a.cx_label = nullptr; a.cx_F = a.cx_T = a.cx_r = a.cx_nvalid = 0; a.cx_scale = nullptr;
  a.cx_lo = nullptr; a.cx_loss = nullptr; a.cx_db = nullptr;
  cudaStream_t st = (cudaStream_t)stream;
#define PASE_NT(BNV)                                                                       \
  switch (mode * 2 + (c_bf16 ? 1 : 0)) {                                                   \
    case 0: return launch_nt<BNV, 0, false, false>(ah, al, bh, bl, a, st);                 \
    case 1: return launch_nt<BNV, 0, true, false>(ah, al, bh, bl, a, st);                  \
    case 2: return launch_nt<BNV, 1, false, false>(ah, al, bh, bl, a, st);                 \
    case 3: return launch_nt<BNV, 1, true, false>(ah, al, bh, bl, a, st);                  \
    case 4: return launch_nt<BNV, 2, false, false>(ah, al, bh, bl, a, st);                 \
    case 5: return launch_nt<BNV, 2, true, false>(ah, al, bh, bl, a, st);                  \
    case 6: return launch_nt<BNV, 3, false, false>(ah, al, bh, bl, a, st);                 \
    default: return launch_nt<BNV, 3, true, false>(ah, al, bh, bl, a, st);                 \
  }
  if (BN == 64) { PASE_NT(64) }
  PASE_NT(128)
#undef PASE_NT
}

// Fused output layer of a regression head (MLPMinion W + ContextualizedLoss MSE,
// minions.py:494-524, losses.py:15-37): residual = A B^T + bias - ctx(label) is never stored
// as fp32; the fp16 pair of s * residual (the backward GEMMs' operand), sum residual^2 and
// the column sums (bias gradient) come out of the GEMM epilogue.  3xF16 operands.
int pase_tc_gemm_nt_ctxmse(const void* Ahi, const void* Alo, long a_rows, int R, const void* Bhi,
                           const void* Blo, long ldb, void* Rhi, void* Rlo, long ldr, int M,
                           int N, int K, const float* bias, const float* label, int B, int F,
                           int T, int r, const float* scale, double* loss_acc, double* db_acc,
                           void* stream) {
  PASE_CHECK_ARG(Ahi && Alo && Bhi && Blo && Rhi && Rlo && label && scale && loss_acc && db_acc,
                 "pase_tc_gemm_nt_ctxmse: null pointer");
  PASE_CHECK_ARG(M == B * T && N == F * r && r >= 1 && (r & 1) && K > 0,
                 "pase_tc_gemm_nt_ctxmse: need M == B*T, N == F*r, odd r (M=%d N=%d)", M, N);
  PASE_CHECK_ARG(R >= 64 && (R % 64) == 0 && (K % 8) == 0 && (ldb % 8) == 0 && ldb >= K,
                 "pase_tc_gemm_nt_ctxmse: operand alignment (R=%d K=%d ldb=%ld)", R, K, ldb);
  PASE_CHECK_ARG((ldr % 128) == 0 && ldr >= N && aligned16(Rhi) && aligned16(Rlo),
                 "pase_tc_gemm_nt_ctxmse: ldr=%ld must be a multiple of 128 and >= N", ldr);
  pase_tc_init_diag();
  const int mode = 3, esz = 2, bk = 64;
  CUtensorMap ah, al, bh, bl;
  uint64_t adims[2] = {(uint64_t)R, (uint64_t)a_rows};
  uint64_t astr[1] = {(uint64_t)R * esz};
  uint32_t abox[2] = {(uint32_t)bk, (uint32_t)BM};
  uint64_t bdims[2] = {(uint64_t)K, (uint64_t)N};          // rows >= N: zero-filled by TMA
  uint64_t bstr[1] = {(uint64_t)ldb * esz};
  uint32_t bbox[2] = {(uint32_t)bk, 128};
  int rc;
  if ((rc = make_map(&ah, Ahi, mode, 2, adims, astr, abox, "ctx A.hi")) != 0) return rc;
  if ((rc = make_map(&al, Alo, mode, 2, adims, astr, abox, "ctx A.lo")) != 0) return rc;
  if ((rc = make_map(&bh, Bhi, mode, 2, bdims, bstr, bbox, "ctx B.hi")) != 0) return rc;
  if ((rc = make_map(&bl, Blo, mode, 2, bdims, bstr, bbox, "ctx B.lo")) != 0) return rc;
  NTArgs a;
  a.R = R; a.C = Rhi; a.ldc = ldr; a.M = M; a.N = (int)ldr; a.K = K; a.alpha = 1.f;
  a.alpha_dev = nullptr; a.bias = bias;
  a.rm = RowMap{M, M, M, 1, (int)ldr};
  a.colsum = nullptr; a.colsumsq = nullptr; a.accumulate = 0;
  a.flush_kb = K > 512 ? 2 : 0;
  a.stages = 0; a.stat_cols = 0;
  a.cx_label = label; a.cx_F = F; a.cx_T = T; a.cx_r = r; a.cx_nvalid = N; a.cx_scale = scale;
  a.cx_lo = Rlo; a.cx_loss = loss_acc; a.cx_db = db_acc;
  return launch_nt<128, 3, false, true>(ah, al, bh, bl, a, (cudaStream_t)stream);
}

// A: groups x [rows_per_group x lda] starting `offA` rows into each group of pitch `pitchA`
// rows (columns 0..I-1 used); B: folded rows of R elements, group pitch `pitchB` rows.
int pase_tc_gemm_tn(const void* Ahi, const void* Alo, long lda, int pitchA, int offA,
                    const void* Bhi, const void* Blo, int R, int pitchB, long b_rows_total,
                    float* C, long ldc, int I, int J, int groups, int rows_per_group, float alpha,
                    const float* alpha_dev, int accumulate, int mode, void* stream) {
  PASE_CHECK_ARG(Ahi && Bhi && C && I > 0 && J > 0 && groups > 0 && rows_per_group > 0,
                 "pase_tc_gemm_tn: bad args");
  PASE_CHECK_ARG(mode >= 0 && mode <= 3, "pase_tc_gemm_tn: mode %d", mode);
  pase_tc_init_diag();
  const bool split = mode == 1 || mode == 3;
  const int esz = mode >= 2 ? 2 : 4;
  const int eb = 128 / esz;
  PASE_CHECK_ARG(!split || (Alo && Blo), "pase_tc_gemm_tn: split modes need lo operands");
  PASE_CHECK_ARG(R >= eb && (R % eb) == 0 && (lda * esz) % 16 == 0 && (I % 4) == 0 &&
                     (J % eb) == 0,
                 "pase_tc_gemm_tn: need R%%%d==0, lda*%d%%16==0, I%%4==0, J%%%d==0 (R=%d lda=%ld "
                 "I=%d J=%d)", eb, esz, eb, R, lda, I, J);
  cudaStream_t st = (cudaStream_t)stream;
  const int BN = J <= 64 ? 64 : 128;
  const int kr = 4 * (32 / esz);                 // reduction rows per stage
  const int flush_ch = split ? (128 / kr > 0 ? 128 / kr : 1) : 0;   // fold every 128 rows
  CUtensorMap ah, al, bh, bl;
  // A as (128 B, rows-in-group, column blocks, groups): the block dimension has the smallest
  // stride after the inner one, so one box brings BM/eb MN-blocks of [kr rows x 128 B]
  uint64_t adims[4] = {(uint64_t)eb, (uint64_t)rows_per_group, (uint64_t)((I + eb - 1) / eb),
                       (uint64_t)groups};
  uint64_t astr[3] = {(uint64_t)lda * esz, 128, (uint64_t)pitchA * lda * esz};
  uint32_t abox[4] = {(uint32_t)eb, (uint32_t)kr, (uint32_t)(BM / eb), 1};
  // B group g covers folded rows [g*pitchB, ...): rows beyond the allocation are zero-filled
  long rows_in_group = b_rows_total - (long)(groups - 1) * pitchB;
  if (rows_in_group > pitchB + (J + R - 1) / R + 1) rows_in_group = pitchB + (J + R - 1) / R + 1;
  const int b_blocked = (R % BN) == 0;
  uint64_t bdims[4] = {(uint64_t)eb, (uint64_t)rows_in_group, (uint64_t)(R / eb),
                       (uint64_t)groups};
  uint64_t bstr[3] = {(uint64_t)R * esz, 128, (uint64_t)pitchB * R * esz};
  uint32_t bbox[4] = {(uint32_t)eb, (uint32_t)kr, (uint32_t)(b_blocked ? BN / eb : 1), 1};
  // NOTE: when I % eb != 0 the last A column block reads up to eb-1 elements past a row's I
  // columns (they only feed output rows >= I, which are never stored); the caller must
  // keep 128 bytes of slack after the last row of A.
  int rc;
  // fp32 stages are transposed in shared memory by the consumers: plain row-major boxes
  const CUtensorMapSwizzle sw = esz == 4 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
  const char* Ah_off = reinterpret_cast<const char*>(Ahi) + (long)offA * lda * esz;
  if ((rc = make_map(&ah, Ah_off, mode, 4, adims, astr, abox, "tn A.hi", sw)) != 0) return rc;
  if ((rc = make_map(&bh, Bhi, mode, 4, bdims, bstr, bbox, "tn B.hi", sw)) != 0) return rc;
  if (split) {
    const char* Al_off = reinterpret_cast<const char*>(Alo) + (long)offA * lda * esz;
    if ((rc = make_map(&al, Al_off, mode, 4, adims, astr, abox, "tn A.lo", sw)) != 0) return rc;
    if ((rc = make_map(&bl, Blo, mode, 4, bdims, bstr, bbox, "tn B.lo", sw)) != 0) return rc;
  } else {
    al = ah;
    bl = bh;
  }
  TNArgs a;
  a.R = R; a.C = C; a.ldc = ldc; a.I = I; a.J = J; a.groups = groups;
  a.rows_per_group = rows_per_group; a.alpha = alpha; a.alpha_dev = alpha_dev;
  a.chunks_per_split = 0; a.flush_ch = flush_ch; a.stages = 0; a.b_blocked = b_blocked;
  a.accumulate = accumulate; a.ws = nullptr;
#define PASE_TN(BNV)                                                      \
  switch (mode) {                                                         \
    case 0: return launch_tn<BNV, 0>(ah, al, bh, bl, a, st);              \
    case 1: return launch_tn<BNV, 1>(ah, al, bh, bl, a, st);              \
    case 2: return launch_tn<BNV, 2>(ah, al, bh, bl, a, st);              \
    default: return launch_tn<BNV, 3>(ah, al, bh, bl, a, st);             \
  }
  if (BN == 64) { PASE_TN(64) }
  PASE_TN(128)
#undef PASE_TN
}

}  // extern "C"
