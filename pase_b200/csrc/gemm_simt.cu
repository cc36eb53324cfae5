// fp32 FFMA implicit-GEMM kernels (exact-fp32 path of the hot loop).
//
//   gemm_nt : C[map(m), n] = alpha * sum_k A[m*lda+k] * B[n*ldb+k] + bias[n]
//             forward conv / transposed conv / dgrad / linear layers.  A may be an
//             overlapping-row view of a padded channel-last activation (lda < K).
//   gemm_tn : C[i,j] += alpha * sum_r A[rowA(r)*lda+i] * B[rowB(r)*ldb+j]
//             weight gradients (split over the reduction; the splits' partial tiles are
//             summed in split order, so the result does not depend on thread scheduling).
//
// 128 x BN x 16 CTA tile, 256 threads, 8 x (BN/16) register tile per thread,
// global->register prefetch of the next k-slab overlapped with the FFMA loop.
#include "common.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 16;
constexpr int NT = 256;
constexpr int APAD = 4;

template <int BN>
struct SmemNT {
  float As[2][BK][BM + APAD];
  float Bs[2][BK][BN + APAD];
};

struct RowMap {
  int rows_in, t_valid, rows_out, fold, cols_per_fold;
  const int* var_tab;              // packed variable-length map (var_row), VAR kernels only
  int var_n;
};

// ------------------------------------------------------------------ NT ----
template <int BN, bool VAR = false>
__global__ void __launch_bounds__(NT, 2)
gemm_nt_kernel(const float* __restrict__ A, long lda, const float* __restrict__ B, long ldb,
               float* __restrict__ C, long ldc, int M, int N, int K, float alpha,
               const float* __restrict__ bias, RowMap rm,
               double* __restrict__ colsum, double* __restrict__ colsumsq, int accumulate) {
  constexpr int TN = BN / 16;           // columns per thread (8 or 4)
  constexpr int BQ = BN / 64;           // float4 B loads per thread (2 or 1)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmemNT<BN>& sm = *reinterpret_cast<SmemNT<BN>*>(smem_raw);

  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * BM;
  const int tx = tid & 15, ty = tid >> 4;

  // loader mapping: 4 threads per row (4 float4 = 16 k), 64 rows per pass
  const int lrow = tid >> 2, lkq = (tid & 3) * 4;

  float4 ra[2], rb[BQ];
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int m = m0 + lrow + h * 64;
      int k = k0 + lkq;
      ra[h] = (m < M && k < K) ? *reinterpret_cast<const float4*>(A + (long)m * lda + k)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int h = 0; h < BQ; ++h) {
      int n = n0 + lrow + h * 64;
      int k = k0 + lkq;
      rb[h] = (n < N && k < K) ? *reinterpret_cast<const float4*>(B + (long)n * ldb + k)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = lrow + h * 64;
      sm.As[buf][lkq + 0][r] = ra[h].x;
      sm.As[buf][lkq + 1][r] = ra[h].y;
      sm.As[buf][lkq + 2][r] = ra[h].z;
      sm.As[buf][lkq + 3][r] = ra[h].w;
    }
#pragma unroll
    for (int h = 0; h < BQ; ++h) {
      int r = lrow + h * 64;
      sm.Bs[buf][lkq + 0][r] = rb[h].x;
      sm.Bs[buf][lkq + 1][r] = rb[h].y;
      sm.Bs[buf][lkq + 2][r] = rb[h].z;
      sm.Bs[buf][lkq + 3][r] = rb[h].w;
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (K + BK - 1) / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&sm.As[buf][k][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&sm.As[buf][k][64 + ty * 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      float4 b0 = *reinterpret_cast<const float4*>(&sm.Bs[buf][k][tx * 4]);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
      if (TN == 8) {
        float4 b1 = *reinterpret_cast<const float4*>(&sm.Bs[buf][k][(BN / 2) + tx * 4]);
        b[TN - 4] = b1.x; b[TN - 3] = b1.y; b[TN - 2] = b1.z; b[TN - 1] = b1.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // ---------------- epilogue ----------------
  const bool want_stats = (colsum != nullptr);
  float csum[TN], csq[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) { csum[j] = 0.f; csq[j] = 0.f; }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
    int u, t_valid;
    long orow;
    if constexpr (VAR) {
      int o;
      if (!var_row(rm.var_tab, rm.var_n, m, o, t_valid, u)) continue;
      orow = o;
    } else {
      const int g = m / rm.rows_in;
      u = m - g * rm.rows_in;
      orow = (long)g * rm.rows_out + u;
      t_valid = rm.t_valid;
    }
#pragma unroll
    for (int jq = 0; jq < TN / 4; ++jq) {
      const int nb = n0 + (jq == 0 ? tx * 4 : (BN / 2) + tx * 4);
      float v[4];
      bool ok[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = nb + j;
        ok[j] = (n < N) && (u * rm.fold + (n / rm.cols_per_fold) < t_valid);
        float x = acc[i][jq * 4 + j] * alpha;
        if (bias != nullptr && n < N) x += bias[n];
        v[j] = x;
      }
      float* cp = C + orow * ldc + nb;
      if (ok[0] && ok[1] && ok[2] && ok[3] && ((ldc & 3) == 0) && ((nb & 3) == 0) &&
          ((reinterpret_cast<uintptr_t>(C) & 15u) == 0)) {
        float4 o;
        if (accumulate) {
          o = *reinterpret_cast<float4*>(cp);
          o.x += v[0]; o.y += v[1]; o.z += v[2]; o.w += v[3];
          v[0] = o.x; v[1] = o.y; v[2] = o.z; v[3] = o.w;
        } else {
          o = make_float4(v[0], v[1], v[2], v[3]);
        }
        *reinterpret_cast<float4*>(cp) = o;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (ok[j]) {
            if (accumulate) v[j] += cp[j];
            cp[j] = v[j];
          }
      }
      if (want_stats) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (ok[j]) {
            csum[jq * 4 + j] += v[j];
            csq[jq * 4 + j] += v[j] * v[j];
          }
      }
    }
  }

  if (want_stats) {
    // reduce over the 16 ty groups through shared memory (reuse the tile storage)
    __syncthreads();
    float* red = reinterpret_cast<float*>(smem_raw);      // [2][16][BN]
#pragma unroll
    for (int jq = 0; jq < TN / 4; ++jq)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = (jq == 0 ? tx * 4 : (BN / 2) + tx * 4) + j;
        red[(0 * 16 + ty) * BN + c] = csum[jq * 4 + j];
        red[(1 * 16 + ty) * BN + c] = csq[jq * 4 + j];
      }
    __syncthreads();
    for (int c = tid; c < 2 * BN; c += NT) {
      const int which = c / BN, col = c - which * BN;
      if (n0 + col >= N) continue;
      double s = 0.0;
#pragma unroll
      for (int r = 0; r < 16; ++r) s += (double)red[(which * 16 + r) * BN + col];
      atomicAdd((which == 0 ? colsum : colsumsq) + n0 + col, s);
    }
  }
}

// ------------------------------------------------------------------ TN ----
struct RedMap {
  int rows_per_group, pitchA, offA, pitchB, offB;
  long total_rows;
};

template <int BN>
struct SmemTN {
  float As[2][BK][BM + APAD];
  float Bs[2][BK][BN + APAD];
};

template <int BN>
__global__ void __launch_bounds__(NT, 2)
gemm_tn_kernel(const float* __restrict__ A, long lda, const float* __restrict__ B, long ldb,
               float* __restrict__ C, long ldc, int I, int J, RedMap rm, float alpha,
               long rows_per_split, int accumulate, float* __restrict__ ws) {
  constexpr int TN = BN / 16;
  constexpr int BQ = BN / 64;            // float4 per thread per 16-row slab: BN*16/4/256
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmemTN<BN>& sm = *reinterpret_cast<SmemTN<BN>*>(smem_raw);
  const int tid = threadIdx.x;
  const int j0 = blockIdx.x * BN;
  const int i0 = blockIdx.y * BM;
  const long r_begin = (long)blockIdx.z * rows_per_split;
  long r_end = r_begin + rows_per_split;
  if (r_end > rm.total_rows) r_end = rm.total_rows;
  if (r_begin >= r_end) return;
  const int tx = tid & 15, ty = tid >> 4;

  // loader: slab of 16 reduction rows; A: 16 x 128 floats = 512 float4 -> 2/thread
  const int a_kr = tid >> 5;             // 0..7 (+8)
  const int a_c4 = (tid & 31) * 4;       // 0..124
  // B: 16 x BN floats -> BQ float4 per thread
  constexpr int BTHR = BN / 4;           // threads per B row (32 or 16)
  const int b_kr = tid / BTHR;           // rows covered per pass: 256/BTHR (8 or 16)
  const int b_c4 = (tid % BTHR) * 4;
  constexpr int BROWS = NT / BTHR;

  float4 ra[2], rb[BQ];
  auto rowsA = [&](long r) -> long {
    long g = r / rm.rows_per_group;
    long u = r - g * rm.rows_per_group;
    return g * rm.pitchA + rm.offA + u;
  };
  auto rowsB = [&](long r) -> long {
    long g = r / rm.rows_per_group;
    long u = r - g * rm.rows_per_group;
    return g * rm.pitchB + rm.offB + u;
  };
  auto load_tiles = [&](long r0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      long r = r0 + a_kr + h * 8;
      int i = i0 + a_c4;
      ra[h] = (r < r_end && i < I) ? *reinterpret_cast<const float4*>(A + rowsA(r) * lda + i)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int h = 0; h < BQ; ++h) {
      long r = r0 + b_kr + h * BROWS;
      int j = j0 + b_c4;
      rb[h] = (r < r_end && j < J) ? *reinterpret_cast<const float4*>(B + rowsB(r) * ldb + j)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float4*>(&sm.As[buf][a_kr + h * 8][a_c4]) = ra[h];
#pragma unroll
    for (int h = 0; h < BQ; ++h)
      *reinterpret_cast<float4*>(&sm.Bs[buf][b_kr + h * BROWS][b_c4]) = rb[h];
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const long nslab = (r_end - r_begin + BK - 1) / BK;
  load_tiles(r_begin);
  store_tiles(0);
  __syncthreads();
  for (long kt = 0; kt < nslab; ++kt) {
    const int buf = (int)(kt & 1);
    if (kt + 1 < nslab) load_tiles(r_begin + (kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&sm.As[buf][k][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&sm.As[buf][k][64 + ty * 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      float4 b0 = *reinterpret_cast<const float4*>(&sm.Bs[buf][k][tx * 4]);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
      if (TN == 8) {
        float4 b1 = *reinterpret_cast<const float4*>(&sm.Bs[buf][k][(BN / 2) + tx * 4]);
        b[TN - 4] = b1.x; b[TN - 3] = b1.y; b[TN - 2] = b1.z; b[TN - 1] = b1.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nslab) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // one split: straight into C (every element has exactly one writer).  Several splits: into
  // this split's partial tile, summed in split order by pase_splitk_reduce
  float* tile = ws == nullptr ? nullptr
      : ws + (((long)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * (BM * BN);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4);
    if (i0 + r >= I) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int c = j < 4 ? tx * 4 + j : (BN / 2) + tx * 4 + (j - 4);
      if (j0 + c >= J) continue;
      const float v = acc[i][j] * alpha;
      if (tile != nullptr) {
        tile[r * BN + c] = v;
      } else {
        float* p = C + (long)(i0 + r) * ldc + j0 + c;
        *p = accumulate ? *p + v : v;
      }
    }
  }
}

template <int BN, bool VAR = false>
int launch_nt(const float* A, long lda, const float* B, long ldb, float* C, long ldc, int M,
              int N, int K, float alpha, const float* bias, RowMap rm, double* colsum,
              double* colsumsq, int accumulate, cudaStream_t st) {
  static bool attr_set = false;
  const size_t smem = sizeof(SmemNT<BN>);
  if (!attr_set) {
    cudaFuncSetAttribute(gemm_nt_kernel<BN, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)smem);
    attr_set = true;
  }
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  gemm_nt_kernel<BN, VAR><<<grid, NT, smem, st>>>(A, lda, B, ldb, C, ldc, M, N, K, alpha, bias, rm,
                                            colsum, colsumsq, accumulate);
  PASE_LAUNCH_CHECK("pase_gemm_nt");
  return PASE_OK;
}

template <int BN>
int launch_tn(const float* A, long lda, const float* B, long ldb, float* C, long ldc, int I,
              int J, RedMap rm, float alpha, int accumulate, cudaStream_t st) {
  static bool attr_set = false;
  const size_t smem = sizeof(SmemTN<BN>);
  if (!attr_set) {
    cudaFuncSetAttribute(gemm_tn_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)smem);
    attr_set = true;
  }
  const int ti = (I + BM - 1) / BM, tj = (J + BN - 1) / BN;
  const long tiles = (long)ti * tj;
  const int target = 3 * pase_num_sms();
  long splits = (target + tiles - 1) / tiles;
  long max_splits = (rm.total_rows + 4 * BK - 1) / (4 * BK);
  if (splits > max_splits) splits = max_splits;
  // the partial tiles must fit the workspace: ceil(3 sms / tiles) * tiles exceeds it for
  // 2 sms < tiles < 3 sms
  if (splits * tiles > pase_splitk_ws_tiles()) splits = pase_splitk_ws_tiles() / tiles;
  if (splits < 1) splits = 1;
  long rps = (rm.total_rows + splits - 1) / splits;
  rps = ((rps + BK - 1) / BK) * BK;
  splits = (rm.total_rows + rps - 1) / rps;     // no empty split
  float* ws = nullptr;
  if (splits > 1 && (ws = pase_splitk_workspace(st, "pase_gemm_tn")) == nullptr)
    return PASE_ERR_UNSUPPORTED;
  dim3 grid(tj, ti, (unsigned)splits);
  gemm_tn_kernel<BN><<<grid, NT, smem, st>>>(A, lda, B, ldb, C, ldc, I, J, rm, alpha, rps,
                                            accumulate, ws);
  PASE_LAUNCH_CHECK("pase_gemm_tn");
  if (splits > 1)
    return pase_splitk_reduce(ws, (int)splits, tj, BN, tiles, C, ldc, I, J, accumulate, st,
                              "pase_gemm_tn");
  return PASE_OK;
}

}  // namespace

extern "C" int pase_gemm_nt(const float* A, long lda, const float* B, long ldb, float* C,
                            long ldc, int M, int N, int K, float alpha, const float* bias,
                            int rows_in, int t_valid, int rows_out, int fold, double* colsum,
                            double* colsumsq, int accumulate, void* stream) {
  PASE_CHECK_ARG(A && B && C, "pase_gemm_nt: null operand");
  PASE_CHECK_ARG(M > 0 && N > 0 && K > 0, "pase_gemm_nt: bad shape M=%d N=%d K=%d", M, N, K);
  PASE_CHECK_ARG((lda % 4) == 0 && (ldb % 4) == 0 && (K % 4) == 0,
                 "pase_gemm_nt: lda, ldb, K must be multiples of 4 (lda=%ld ldb=%ld K=%d)", lda,
                 ldb, K);
  PASE_CHECK_ARG(aligned16(A) && aligned16(B), "pase_gemm_nt: A/B must be 16-byte aligned");
  PASE_CHECK_ARG(rows_in > 0 && rows_out > 0 && fold > 0 && (N % fold) == 0,
                 "pase_gemm_nt: bad row map rows_in=%d rows_out=%d fold=%d N=%d", rows_in,
                 rows_out, fold, N);
  PASE_CHECK_ARG((colsum == nullptr) == (colsumsq == nullptr),
                 "pase_gemm_nt: colsum and colsumsq must be given together");
  RowMap rm{rows_in, t_valid, rows_out, fold, N / fold, nullptr, 0};
  cudaStream_t st = (cudaStream_t)stream;
  if (N <= 64)
    return launch_nt<64>(A, lda, B, ldb, C, ldc, M, N, K, alpha, bias, rm, colsum, colsumsq,
                         accumulate, st);
  return launch_nt<128>(A, lda, B, ldb, C, ldc, M, N, K, alpha, bias, rm, colsum, colsumsq,
                        accumulate, st);
}

extern "C" int pase_gemm_tn(const float* A, long lda, int pitchA, int offA, const float* B,
                            long ldb, int pitchB, int offB, float* C, long ldc, int I, int J,
                            int groups, int rows_per_group, float alpha, int accumulate,
                            void* stream) {
  PASE_CHECK_ARG(A && B && C, "pase_gemm_tn: null operand");
  PASE_CHECK_ARG(I > 0 && J > 0 && groups > 0 && rows_per_group > 0,
                 "pase_gemm_tn: bad shape I=%d J=%d groups=%d rows=%d", I, J, groups,
                 rows_per_group);
  PASE_CHECK_ARG((lda % 4) == 0 && (ldb % 4) == 0 && (I % 4) == 0 && (J % 4) == 0,
                 "pase_gemm_tn: lda, ldb, I, J must be multiples of 4 (lda=%ld ldb=%ld I=%d J=%d)",
                 lda, ldb, I, J);
  PASE_CHECK_ARG(aligned16(A) && aligned16(B), "pase_gemm_tn: A/B must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  RedMap rm{rows_per_group, pitchA, offA, pitchB, offB, (long)groups * rows_per_group};
  if (J <= 64) return launch_tn<64>(A, lda, B, ldb, C, ldc, I, J, rm, alpha, accumulate, st);
  return launch_tn<128>(A, lda, B, ldb, C, ldc, I, J, rm, alpha, accumulate, st);
}

// pase_gemm_nt_var and pase_gemm_nt_var_stats (colsum / colsumsq NULL: no statistics)
static int gemm_nt_var_impl(const char* fn, const float* A, long lda, const float* B, long ldb,
                            float* C, long ldc, int M, int N, int K, const float* bias,
                            const int* var_tab, int nvar, int fold, double* colsum,
                            double* colsumsq, void* stream) {
  PASE_CHECK_ARG(A && B && C && var_tab && nvar > 0, "%s: null operand / table", fn);
  PASE_CHECK_ARG(M > 0 && N > 0 && K > 0, "%s: bad shape M=%d N=%d K=%d", fn, M, N, K);
  PASE_CHECK_ARG((lda % 4) == 0 && (ldb % 4) == 0 && (K % 4) == 0,
                 "%s: lda, ldb, K must be multiples of 4 (lda=%ld ldb=%ld K=%d)", fn, lda, ldb, K);
  PASE_CHECK_ARG(aligned16(A) && aligned16(B), "%s: A/B must be 16-byte aligned", fn);
  PASE_CHECK_ARG(fold > 0 && (N % fold) == 0, "%s: fold=%d N=%d", fn, fold, N);
  RowMap rm{1, 0, 1, fold, N / fold, var_tab, nvar};
  cudaStream_t st = (cudaStream_t)stream;
  if (N <= 64)
    return launch_nt<64, true>(A, lda, B, ldb, C, ldc, M, N, K, 1.f, bias, rm, colsum, colsumsq,
                               0, st);
  return launch_nt<128, true>(A, lda, B, ldb, C, ldc, M, N, K, 1.f, bias, rm, colsum, colsumsq, 0,
                              st);
}

extern "C" int pase_gemm_nt_var(const float* A, long lda, const float* B, long ldb, float* C,
                                long ldc, int M, int N, int K, const float* bias,
                                const int* var_tab, int nvar, int fold, void* stream) {
  return gemm_nt_var_impl("pase_gemm_nt_var", A, lda, B, ldb, C, ldc, M, N, K, bias, var_tab,
                          nvar, fold, nullptr, nullptr, stream);
}

extern "C" int pase_gemm_nt_var_stats(const float* A, long lda, const float* B, long ldb,
                                      float* C, long ldc, int M, int N, int K, const float* bias,
                                      const int* var_tab, int nvar, int fold, double* colsum,
                                      double* colsumsq, void* stream) {
  PASE_CHECK_ARG(colsum && colsumsq, "pase_gemm_nt_var_stats: null statistics");
  return gemm_nt_var_impl("pase_gemm_nt_var_stats", A, lda, B, ldb, C, ldc, M, N, K, bias,
                          var_tab, nvar, fold, colsum, colsumsq, stream);
}
