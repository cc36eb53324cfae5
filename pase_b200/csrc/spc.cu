// SPC worker frame gather (SPCMinion, minions.py:575-649 of the reference) with the three frame
// indices read from a device table, so the draws of a captured training step can change from one
// replay to the next.
//
//   pase_spc_gather      (2B, (N+1)C) rows [cur | fut ; cur | past] from the encoder's
//                        channel-last rows, fut / past flattened channel-major (c * N + n)
//   pase_spc_gather_bwd  the dense (B*T, C) gradient: the windows copied, the two cur halves
//                        summed at frame t, zeros elsewhere; no atomics
//
// The host (pase_b200/functional.py) validates the indices before they are uploaded:
// M + 1 <= t < T - M, t + seq_pad <= future_t < T - N, N <= past_t < t - seq_pad (M = seq_pad + N),
// so the kernels trust the table.
#include <algorithm>
#include "common.cuh"

namespace {

constexpr int SPC_THREADS = 256;
constexpr int MAX_B = 65535;

__global__ void __launch_bounds__(SPC_THREADS)
spc_gather_kernel(const float* __restrict__ x, long ldx, const long* __restrict__ frames, int B,
                  int T, int C, int N, float* __restrict__ out) {
  pdl_wait();
  const int r = blockIdx.x;                       // output row: b (pos) or B + b (neg)
  const bool neg = r >= B;
  const int b = neg ? r - B : r;
  const long t = frames[0];
  const long w0 = neg ? frames[2] - N : frames[1];          // first frame of the window
  const long base = (long)b * T;
  const int W = (N + 1) * C;
  float* o = out + (long)r * W;
  for (int j = threadIdx.x; j < W; j += blockDim.x) {
    long src;
    if (j < C) {
      src = (base + t) * ldx + j;
    } else {
      const int k = j - C, c = k / N, n = k - c * N;
      src = (base + w0 + n) * ldx + c;
    }
    o[j] = x[src];
  }
}

__global__ void __launch_bounds__(SPC_THREADS)
spc_gather_bwd_kernel(const float* __restrict__ g, const long* __restrict__ frames, int B, int T,
                      int C, int N, float* __restrict__ dx) {
  pdl_wait();
  const long t = frames[0], ft = frames[1], p0 = frames[2] - N;
  const long W = (long)(N + 1) * C;
  const long total = (long)B * T * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const long row = i / C;
    const int c = (int)(i - row * C);
    const long b = row / T, f = row - b * T;
    const float* gp = g + b * W;                  // [cur | fut] row of sample b
    const float* gn = g + (B + b) * W;            // [cur | past] row
    float v = 0.f;
    // autograd of the torch gather: cur's two uses are summed first, then the view's inputs
    // (only the fut window can meet frame t, when seq_pad = 0)
    if (f == t) v = gp[c] + gn[c];
    if (f >= ft && f < ft + N) v += gp[C + (long)c * N + (f - ft)];
    else if (f >= p0 && f < p0 + N) v = gn[C + (long)c * N + (f - p0)];
    dx[i] = v;
  }
}

}  // namespace

extern "C" {

int pase_spc_gather(const float* x, long ldx, const long* frames, int B, int T, int C, int N,
                    int seq_pad, float* out, void* stream) {
  PASE_CHECK_ARG(x, "pase_spc_gather: x is NULL");
  PASE_CHECK_ARG(frames, "pase_spc_gather: frames is NULL");
  PASE_CHECK_ARG(out, "pase_spc_gather: out is NULL");
  PASE_CHECK_ARG(B > 0 && B <= MAX_B, "pase_spc_gather: B=%d outside [1, %d]", B, MAX_B);
  PASE_CHECK_ARG(C > 0, "pase_spc_gather: C=%d", C);
  PASE_CHECK_ARG(N >= 0 && seq_pad >= 0, "pase_spc_gather: N=%d seq_pad=%d", N, seq_pad);
  PASE_CHECK_ARG((long)(N + 1) * C <= (1L << 24), "pase_spc_gather: (N+1)*C=%ld",
                 (long)(N + 1) * C);
  PASE_CHECK_ARG(ldx >= C, "pase_spc_gather: ldx=%ld < C=%d", ldx, C);
  // the current frame's range [M + 1, T - M) must not be empty
  PASE_CHECK_ARG((long)T - (seq_pad + N) > (long)seq_pad + N + 1,
                 "pase_spc_gather: T=%d frames leave no current frame for N=%d seq_pad=%d", T, N,
                 seq_pad);
  PASE_LAUNCH((spc_gather_kernel), 2 * B, SPC_THREADS, 0, (cudaStream_t)stream, x, ldx, frames, B,
              T, C, N, out);
  PASE_LAUNCH_CHECK("pase_spc_gather");
  return PASE_OK;
}

int pase_spc_gather_bwd(const float* g, const long* frames, int B, int T, int C, int N,
                        int seq_pad, float* dx, void* stream) {
  PASE_CHECK_ARG(g, "pase_spc_gather_bwd: g is NULL");
  PASE_CHECK_ARG(frames, "pase_spc_gather_bwd: frames is NULL");
  PASE_CHECK_ARG(dx, "pase_spc_gather_bwd: dx is NULL");
  PASE_CHECK_ARG(B > 0 && B <= MAX_B, "pase_spc_gather_bwd: B=%d outside [1, %d]", B, MAX_B);
  PASE_CHECK_ARG(C > 0, "pase_spc_gather_bwd: C=%d", C);
  PASE_CHECK_ARG(N >= 0 && seq_pad >= 0, "pase_spc_gather_bwd: N=%d seq_pad=%d", N, seq_pad);
  PASE_CHECK_ARG((long)(N + 1) * C <= (1L << 24), "pase_spc_gather_bwd: (N+1)*C=%ld",
                 (long)(N + 1) * C);
  PASE_CHECK_ARG((long)T - (seq_pad + N) > (long)seq_pad + N + 1,
                 "pase_spc_gather_bwd: T=%d frames leave no current frame for N=%d seq_pad=%d", T,
                 N, seq_pad);
  const long total = (long)B * T * C;
  const int blocks = (int)std::min<long>((total + SPC_THREADS - 1) / SPC_THREADS, 1184);
  PASE_LAUNCH((spc_gather_bwd_kernel), blocks, SPC_THREADS, 0, (cudaStream_t)stream, g, frames, B,
              T, C, N, dx);
  PASE_LAUNCH_CHECK("pase_spc_gather_bwd");
  return PASE_OK;
}

}  // extern "C"
