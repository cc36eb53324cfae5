// Worker-head losses, fused with their label handling:
//   contextualised MSE (losses.py:15-37 + nn.MSELoss) without materialising the
//   r-times unfolded label; L1 (cchunk decoder); BCE-with-logits against the
//   [ones; zeros] pair labels of LIM/GIM (cls_minions.py:47-51); GIM time mean.
#include "common.cuh"

namespace {

constexpr int TPB = 256;

__device__ __forceinline__ void block_acc(double v, double* acc) {
  __shared__ double wsum[TPB / 32];
  v = warp_sum_d(v);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) wsum[w] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < TPB / 32; ++i) s += wsum[i];
    atomicAdd(acc, s);
  }
}

// Thread = one prediction column (f, j fixed: no per-element divisions), block = 256 columns
// x CTX_RPB rows: pred is read coalesced along the columns, the label window
// label[b][f][t + j - r/2] walks contiguously in t (L1-resident: every label element serves r
// predictions).  HBM-bound: 4 B (fwd) / 8 B (bwd) per prediction element.
constexpr int CTX_RPB = 32;

__global__ void __launch_bounds__(TPB)
ctx_mse_fwd_kernel(const float* __restrict__ pred, long ldp, const float* __restrict__ label,
                   long rows, int F, int T, int r, double* acc) {
  const int cols = F * r;
  const int col = blockIdx.x * TPB + threadIdx.x;
  const long row0 = (long)blockIdx.y * CTX_RPB;
  float s = 0.f;
  if (col < cols) {
    const int f = col / r, shift = (col - f * r) - r / 2;
    long b = row0 / T;
    int t = (int)(row0 - b * T);
    const float* p = pred + row0 * ldp + col;
    const int n = (rows - row0) < CTX_RPB ? (int)(rows - row0) : CTX_RPB;
#pragma unroll 4
    for (int i = 0; i < n; ++i) {
      const int tt = t + shift;
      const float lab = (tt >= 0 && tt < T) ? __ldg(label + (b * F + f) * T + tt) : 0.f;
      const float d = p[(long)i * ldp] - lab;
      s = fmaf(d, d, s);
      if (++t == T) { t = 0; ++b; }
    }
  }
  block_acc((double)s, acc);
}

__global__ void __launch_bounds__(TPB)
ctx_mse_bwd_kernel(const float* __restrict__ pred, long ldp, const float* __restrict__ label,
                   long rows, int F, int T, int r, float coef, const float* __restrict__ gscale,
                   float* __restrict__ dpred, long lddp) {
  const int cols = F * r;
  const int col = blockIdx.x * TPB + threadIdx.x;
  if (col >= cols) return;
  const long row0 = (long)blockIdx.y * CTX_RPB;
  const float k = coef * (gscale ? gscale[0] : 1.f);
  const int f = col / r, shift = (col - f * r) - r / 2;
  long b = row0 / T;
  int t = (int)(row0 - b * T);
  const float* p = pred + row0 * ldp + col;
  float* dp = dpred + row0 * lddp + col;
  const int n = (rows - row0) < CTX_RPB ? (int)(rows - row0) : CTX_RPB;
#pragma unroll 4
  for (int i = 0; i < n; ++i) {
    const int tt = t + shift;
    const float lab = (tt >= 0 && tt < T) ? __ldg(label + (b * F + f) * T + tt) : 0.f;
    dp[(long)i * lddp] = k * (p[(long)i * ldp] - lab);
    if (++t == T) { t = 0; ++b; }
  }
}

__global__ void __launch_bounds__(TPB)
l1_fwd_kernel(const float* __restrict__ p, const float* __restrict__ t, long n, double* acc) {
  double s = 0.0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long)gridDim.x * blockDim.x)
    s += (double)fabsf(p[i] - t[i]);
  block_acc(s, acc);
}

__global__ void l1_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t, long n,
                              float coef, const float* __restrict__ gscale,
                              float* __restrict__ dp) {
  const float k = coef * (gscale ? gscale[0] : 1.f);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long)gridDim.x * blockDim.x) {
    const float d = p[i] - t[i];
    dp[i] = d > 0.f ? k : (d < 0.f ? -k : 0.f);
  }
}

__global__ void __launch_bounds__(TPB)
bce_pairs_fwd_kernel(const float* __restrict__ x, long n, long n_pos, double* acc) {
  double s = 0.0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float y = i < n_pos ? 1.f : 0.f;
    // max(v, 0) - v y + log(1 + e^-|v|): for a confident logit the first two terms cancel
    // exactly and log1pf keeps the e^-|v| that log(1 + e^-|v|) rounds away above |v| ~ 17
    s += (double)(fmaxf(v, 0.f) - v * y + log1pf(expf(-fabsf(v))));
  }
  block_acc(s, acc);
}

__global__ void bce_pairs_bwd_kernel(const float* __restrict__ x, long n, long n_pos, float coef,
                                     const float* __restrict__ gscale, float* __restrict__ dx) {
  const float k = coef * (gscale ? gscale[0] : 1.f);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float y = i < n_pos ? 1.f : 0.f;
    dx[i] = k * (1.f / (1.f + expf(-v)) - y);
  }
}

// x (B, T, *) row stride ldx -> out (B, C): mean over T
__global__ void time_mean_fwd_kernel(const float* __restrict__ x, long ldx, float* __restrict__ out,
                                     long ldo, int T, int C) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int t = 0; t < T; ++t) s += x[((long)b * T + t) * ldx + c];
  out[(long)b * ldo + c] = s / (float)T;
}

__global__ void time_mean_bwd_kernel(const float* __restrict__ dout, long ldo,
                                     float* __restrict__ dx, long ldx, int T, int C,
                                     int accumulate) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float g = dout[(long)b * ldo + c] / (float)T;
  for (int t = 0; t < T; ++t) {
    float* p = dx + ((long)b * T + t) * ldx + c;
    *p = accumulate ? *p + g : g;
  }
}

inline unsigned nblk(long total) {
  long b = (total + TPB - 1) / TPB;
  long cap = (long)pase_num_sms() * 8;
  return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" {

int pase_ctx_mse_fwd(const float* pred, long ldp, const float* label, int B, int F, int T, int r,
                     double* acc, void* stream) {
  PASE_CHECK_ARG(pred && label && acc && B > 0 && F > 0 && T > 0 && r >= 1 && (r & 1),
                 "pase_ctx_mse_fwd: bad args (r must be odd, got %d)", r);
  const long rows = (long)B * T;
  const dim3 cgrid((unsigned)((F * r + TPB - 1) / TPB), (unsigned)((rows + CTX_RPB - 1) / CTX_RPB));
  ctx_mse_fwd_kernel<<<cgrid, TPB, 0, (cudaStream_t)stream>>>(pred, ldp, label, rows,
                                                                          F, T, r, acc);
  PASE_LAUNCH_CHECK("pase_ctx_mse_fwd");
  return PASE_OK;
}

int pase_ctx_mse_bwd(const float* pred, long ldp, const float* label, int B, int F, int T, int r,
                     float coef, const float* gscale, float* dpred, long lddp, void* stream) {
  PASE_CHECK_ARG(pred && label && dpred && B > 0 && F > 0 && T > 0 && r >= 1 && (r & 1),
                 "pase_ctx_mse_bwd: bad args");
  const long rows = (long)B * T;
  const dim3 cgrid((unsigned)((F * r + TPB - 1) / TPB), (unsigned)((rows + CTX_RPB - 1) / CTX_RPB));
  ctx_mse_bwd_kernel<<<cgrid, TPB, 0, (cudaStream_t)stream>>>(
      pred, ldp, label, rows, F, T, r, coef, gscale, dpred, lddp);
  PASE_LAUNCH_CHECK("pase_ctx_mse_bwd");
  return PASE_OK;
}

int pase_l1_fwd(const float* pred, const float* target, long n, double* acc, void* stream) {
  PASE_CHECK_ARG(pred && target && acc && n > 0, "pase_l1_fwd: bad args");
  l1_fwd_kernel<<<nblk(n), TPB, 0, (cudaStream_t)stream>>>(pred, target, n, acc);
  PASE_LAUNCH_CHECK("pase_l1_fwd");
  return PASE_OK;
}

int pase_l1_bwd(const float* pred, const float* target, long n, float coef, const float* gscale,
                float* dpred, void* stream) {
  PASE_CHECK_ARG(pred && target && dpred && n > 0, "pase_l1_bwd: bad args");
  l1_bwd_kernel<<<nblk(n), TPB, 0, (cudaStream_t)stream>>>(pred, target, n, coef, gscale, dpred);
  PASE_LAUNCH_CHECK("pase_l1_bwd");
  return PASE_OK;
}

int pase_bce_pairs_fwd(const float* logit, long n, long n_pos, double* acc, void* stream) {
  PASE_CHECK_ARG(logit && acc && n > 0 && n_pos >= 0 && n_pos <= n, "pase_bce_pairs_fwd: bad args");
  bce_pairs_fwd_kernel<<<nblk(n), TPB, 0, (cudaStream_t)stream>>>(logit, n, n_pos, acc);
  PASE_LAUNCH_CHECK("pase_bce_pairs_fwd");
  return PASE_OK;
}

int pase_bce_pairs_bwd(const float* logit, long n, long n_pos, float coef, const float* gscale,
                       float* dlogit, void* stream) {
  PASE_CHECK_ARG(logit && dlogit && n > 0 && n_pos >= 0 && n_pos <= n,
                 "pase_bce_pairs_bwd: bad args");
  bce_pairs_bwd_kernel<<<nblk(n), TPB, 0, (cudaStream_t)stream>>>(logit, n, n_pos, coef, gscale,
                                                                 dlogit);
  PASE_LAUNCH_CHECK("pase_bce_pairs_bwd");
  return PASE_OK;
}

int pase_time_mean_fwd(const float* x, long ldx, float* out, long ldo, int B, int T, int C,
                       void* stream) {
  PASE_CHECK_ARG(x && out && B > 0 && T > 0 && C > 0, "pase_time_mean_fwd: bad args");
  dim3 grid((C + 127) / 128, B);
  time_mean_fwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(x, ldx, out, ldo, T, C);
  PASE_LAUNCH_CHECK("pase_time_mean_fwd");
  return PASE_OK;
}

int pase_time_mean_bwd(const float* dout, long ldo, float* dx, long ldx, int B, int T, int C,
                       int accumulate, void* stream) {
  PASE_CHECK_ARG(dout && dx && B > 0 && T > 0 && C > 0, "pase_time_mean_bwd: bad args");
  dim3 grid((C + 127) / 128, B);
  time_mean_bwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(dout, ldo, dx, ldx, T, C,
                                                               accumulate);
  PASE_LAUNCH_CHECK("pase_time_mean_bwd");
  return PASE_OK;
}

}  // extern "C"
