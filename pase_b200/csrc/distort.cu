// On-device waveform DISTORTIONS (SURVEY.md 8f, row N3): the PASE+ stages of
// pase/transforms.py:38-146 config_distortions / PCompose whose arithmetic is numpy/scipy --
// Reverb (transforms.py:1001-1103), SimpleAdditiveShift (1684-1766), SimpleAdditive
// (1576-1675), Clipping (1514-1536), BandDrop (1207-1297) and Downsample (1113-1197).  The
// reference runs them per sample on DataLoader workers with scipy; here they run on a collated
// batch in HBM.  The host draws a per-sample plan (pase_b200/distortions.py); every kernel reads
// which samples it touches from a device job table, so launch shapes depend only on
// (jobs, T, longest filter) and the pipeline can be captured in a CUDA graph.
//
//   pase_fft_conv        signal.convolve(x, h, 'full') restricted to the window [p, p+n), and
//                        the energy the stage normalises with, as uniformly partitioned
//                        overlap-save: 4096-sample blocks, 8192-point complex fp32 FFTs in shared
//                        memory, then the energy scale of the Reverb / FIR stages
//   pase_segment_gather  noise / overlap segment from the device noise pool, zero-padded
//   pase_noise_mix       SimpleAdditive / SimpleAdditiveShift mix + energy normalisation
//   pase_clip            Clipping
//   pase_overlap_label   the overlap label of SimpleAdditiveShift, window-averaged
//
// Every per-sample reduction is fp64 in a fixed order (per-thread strided sums, a shuffle
// tree, then the warps in index order), so two runs give equal bits.
#include <algorithm>
#include "common.cuh"

namespace {

constexpr int FFT_LOG = 13;
constexpr int FFT_N = 1 << FFT_LOG;     // 8192-point transforms
constexpr int BLK = FFT_N / 2;          // 4096-sample blocks and filter partitions
constexpr int FFT_THREADS = 512;
constexpr int RED_THREADS = 512;
constexpr size_t FFT_SMEM = (size_t)FFT_N * sizeof(float2);   // 64 KB

// conv job row: {on, n, filt_off, L, p, mode}
constexpr int CJ = 6;
// mode 0: FIR (BandDrop / Downsample): energy of the trimmed window; E == 0 keeps x
// mode 1: Reverb: energy of the full convolution (length n + L - 1); E == 0 scales by 1
// mode 2: raw window, no scaling
struct ConvJob {
  long n, off, L, p, mode;
  bool on;
};

__device__ __forceinline__ ConvJob load_job(const long* jobs, int b, int T, int Lmax, long bank_len) {
  const long* r = jobs + (long)b * CJ;
  ConvJob j;
  j.n = r[1]; j.off = r[2]; j.L = r[3]; j.p = r[4]; j.mode = r[5];
  // a malformed row is treated as "not drawn" rather than read out of bounds
  j.on = r[0] != 0 && j.n > 0 && j.n <= T && j.L > 0 && j.L <= Lmax && j.p >= 0 && j.p < j.L &&
         j.off >= 0 && j.off + j.L <= bank_len && j.mode >= 0 && j.mode <= 2;
  return j;
}
__device__ __forceinline__ int job_blocks(const ConvJob& j) { return (int)((j.n + j.L - 1 + BLK - 1) / BLK); }
__device__ __forceinline__ int job_parts(const ConvJob& j) { return (int)((j.L + BLK - 1) / BLK); }

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// In-place radix-2 decimation-in-time transform of z (loaded in bit-reversed order), natural
// order out.  tw[k] = exp(-2 pi i k / FFT_N), k < FFT_N/2 (fp64 on the host, stored fp32);
// `inv` conjugates the twiddles (the 1/N is the caller's).
__device__ void fft8192(float2* z, const float2* __restrict__ tw, bool inv) {
  __syncthreads();
  for (int s = 0; s < FFT_LOG; ++s) {
    const int h = 1 << s;
    const int tsh = FFT_LOG - 1 - s;          // twiddle stride = N / (2h)
    for (int j = threadIdx.x; j < FFT_N / 2; j += blockDim.x) {
      const int pos = j & (h - 1);
      const int i0 = ((j - pos) << 1) + pos, i1 = i0 + h;
      float2 w = __ldg(tw + (pos << tsh));
      if (inv) w.y = -w.y;
      const float2 a = z[i0], bw = cmul(z[i1], w);
      z[i0] = make_float2(a.x + bw.x, a.y + bw.y);
      z[i1] = make_float2(a.x - bw.x, a.y - bw.y);
    }
    __syncthreads();
  }
}

__device__ __forceinline__ int bitrev(int i) { return (int)(__brev((unsigned)i) >> (32 - FFT_LOG)); }

// fp64 block sum in a fixed order; every thread gets the result
template <int NV>
__device__ void block_sum_d(double (&v)[NV]) {
  __shared__ double red[32][NV];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = warp_sum_d(v[q]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) red[w][q] = v[q];
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    double s = 0.0;
    for (int i = 0; i < nw; ++i) s += red[i][q];
    v[q] = s;
  }
  __syncthreads();
}

// Spectra: CTA (slot, b).  slot < nbmax: X_m of job b, the FFT of x[(m-1)*BLK, (m+1)*BLK)
// (zero outside [0, n)); slot >= nbmax: H_k, the FFT of taps [k*BLK, (k+1)*BLK) zero-padded.
__global__ void __launch_bounds__(FFT_THREADS)
conv_spectra_kernel(const float* __restrict__ x, long ldx, const float* __restrict__ bank,
                    long bank_len, const long* __restrict__ jobs, int T, int Lmax, int nbmax,
                    int pmax, const float2* __restrict__ tw, float2* __restrict__ xspec,
                    float2* __restrict__ hspec) {
  pdl_wait();
  extern __shared__ float2 z[];
  const int b = blockIdx.y, slot = blockIdx.x;
  const ConvJob jb = load_job(jobs, b, T, Lmax, bank_len);
  if (!jb.on) return;
  float2* dst;
  if (slot < nbmax) {
    const int m = slot;
    if (m >= job_blocks(jb)) return;
    const float* xr = x + (long)b * ldx;
    const long base = (long)(m - 1) * BLK;
    for (int j = threadIdx.x; j < FFT_N; j += blockDim.x) {
      const long t = base + j;
      z[bitrev(j)] = make_float2(t >= 0 && t < jb.n ? xr[t] : 0.f, 0.f);
    }
    dst = xspec + ((long)b * nbmax + m) * FFT_N;
  } else {
    const int k = slot - nbmax;
    if (k >= job_parts(jb)) return;
    const float* hr = bank + jb.off;
    for (int j = threadIdx.x; j < FFT_N; j += blockDim.x) {
      const long l = (long)k * BLK + j;
      z[bitrev(j)] = make_float2(j < BLK && l < jb.L ? hr[l] : 0.f, 0.f);
    }
    dst = hspec + ((long)b * pmax + k) * FFT_N;
  }
  fft8192(z, tw, false);
  for (int i = threadIdx.x; i < FFT_N; i += blockDim.x) dst[i] = z[i];
}

// Output block m of job b: Y_m = sum_k X_{m-k} H_k (k ascending), inverse FFT; the last BLK
// samples are the full convolution at [m*BLK, (m+1)*BLK).  Stores the window [p, p+n) into y
// (row stride T) and the block's fp64 energy partial over the stage's energy window.
__global__ void __launch_bounds__(FFT_THREADS)
conv_output_kernel(const long* __restrict__ jobs, int T, int Lmax, long bank_len, int nbmax,
                   int pmax, const float2* __restrict__ tw, const float2* __restrict__ xspec,
                   const float2* __restrict__ hspec, float* __restrict__ y,
                   double* __restrict__ epart) {
  pdl_wait();
  extern __shared__ float2 z[];
  const int b = blockIdx.y, m = blockIdx.x;
  const ConvJob jb = load_job(jobs, b, T, Lmax, bank_len);
  if (!jb.on || m >= job_blocks(jb)) return;
  const int P = job_parts(jb);
  const int kmax = min(P - 1, m);
  const float2* xs = xspec + (long)b * nbmax * FFT_N;
  const float2* hs = hspec + (long)b * pmax * FFT_N;
  for (int i = threadIdx.x; i < FFT_N; i += blockDim.x) {
    float2 acc = make_float2(0.f, 0.f);
    for (int k = 0; k <= kmax; ++k) {
      const float2 a = xs[(long)(m - k) * FFT_N + i], h = hs[(long)k * FFT_N + i];
      acc.x = fmaf(a.x, h.x, fmaf(-a.y, h.y, acc.x));
      acc.y = fmaf(a.x, h.y, fmaf(a.y, h.x, acc.y));
    }
    z[bitrev(i)] = acc;
  }
  fft8192(z, tw, true);
  const float inv_n = 1.f / FFT_N;                      // exact power of two
  const long full = jb.n + jb.L - 1;
  double e[1] = {0.0};
  float* yr = y + (long)b * T;
  for (int j = threadIdx.x; j < BLK; j += blockDim.x) {
    const long i = (long)m * BLK + j;
    const float v = z[BLK + j].x * inv_n;
    const bool in_win = i >= jb.p && i < jb.p + jb.n;
    if (in_win) yr[i - jb.p] = v;
    if (jb.mode == 1 ? i < full : in_win) e[0] += (double)v * v;
  }
  block_sum_d<1>(e);
  if (threadIdx.x == 0) epart[(long)b * nbmax + m] = e[0];
}

// Energy scale of job b, in place when out == x: Ex over x[0, n), E = the partials in block
// order, then out = sqrt(Ex/E) * y (mode 0: x when E == 0; mode 1: y when E == 0; mode 2: y).
__global__ void __launch_bounds__(RED_THREADS)
conv_scale_kernel(const float* x, long ldx, const long* __restrict__ jobs, int T, int Lmax,
                  long bank_len, int nbmax, const float* __restrict__ y,
                  const double* __restrict__ epart, float* out, long ldo) {
  pdl_wait();
  const int b = blockIdx.x;
  const ConvJob jb = load_job(jobs, b, T, Lmax, bank_len);
  if (!jb.on) return;
  const float* xr = x + (long)b * ldx;
  const float* yr = y + (long)b * T;
  float* o = out + (long)b * ldo;
  double ex[1] = {0.0};
  for (long t = threadIdx.x; t < jb.n; t += blockDim.x) ex[0] += (double)xr[t] * xr[t];
  block_sum_d<1>(ex);
  double E = 0.0;
  const int nb = job_blocks(jb);
  for (int m = 0; m < nb; ++m) E += epart[(long)b * nbmax + m];
  const bool keep_x = jb.mode == 0 && !(E > 0.0);
  const float s = (jb.mode == 2 || !(E > 0.0)) ? 1.f : (float)sqrt(ex[0] / E);
  for (long t = threadIdx.x; t < jb.n; t += blockDim.x) o[t] = keep_x ? xr[t] : s * yr[t];
}

// gather job row: {on, pool_off, avail}: out[u] = pool[pool_off + u] for u < avail, 0 for
// avail <= u < T
__global__ void segment_gather_kernel(const float* __restrict__ pool, long pool_len,
                                      const long* __restrict__ jobs, int T,
                                      float* __restrict__ out, long ldo) {
  pdl_wait();
  const int b = blockIdx.y;
  const long* r = jobs + (long)b * 3;
  const long off = r[1], avail = r[2];
  if (r[0] == 0 || off < 0 || avail < 0 || avail > T || off + avail > pool_len) return;
  float* o = out + (long)b * ldo;
  for (long u = (long)blockIdx.x * blockDim.x + threadIdx.x; u < T; u += (long)gridDim.x * blockDim.x)
    o[u] = u < avail ? pool[off + u] : 0.f;
}

// mix job row: {on, shift, guard}; n[t] = 0 for t < shift, seg[t - shift] after.
// K = sqrt(Ex / (snr_lin En)) (1 when En == 0), v = x + K n, x <- sqrt(Ex / (v.v + 1e-14)) v;
// v.v = Ex + 2K Exn + K^2 En from the same pass.  guard: En == 0 leaves x unchanged.
__global__ void __launch_bounds__(RED_THREADS)
noise_mix_kernel(float* x, long ldx, const float* __restrict__ seg, long lds,
                 const long* __restrict__ jobs, const double* __restrict__ snr_lin, int T) {
  pdl_wait();
  const int b = blockIdx.x;
  const long* r = jobs + (long)b * 3;
  const long shift = r[1];
  if (r[0] == 0 || shift < 0 || shift >= T) return;
  float* xr = x + (long)b * ldx;
  const float* sr = seg + (long)b * lds - shift;
  double v[3] = {0.0, 0.0, 0.0};                   // Ex, En, Exn
  for (long t = threadIdx.x; t < T; t += blockDim.x) {
    const double a = xr[t], n = t >= shift ? (double)sr[t] : 0.0;
    v[0] += a * a;
    v[1] += n * n;
    v[2] += a * n;
  }
  block_sum_d<3>(v);
  const double Ex = v[0], En = v[1], Exn = v[2];
  if (r[2] != 0 && !(En > 0.0)) return;
  const double K = En > 0.0 ? sqrt(Ex / (snr_lin[b] * En)) : 1.0;
  const double Ev = Ex + 2.0 * K * Exn + K * K * En;
  const float g = (float)sqrt(Ex / (Ev + 1e-14)), Kf = (float)K;
  for (long t = threadIdx.x; t < T; t += blockDim.x) {
    const float n = t >= shift ? sr[t] : 0.f;
    xr[t] = g * (xr[t] + Kf * n);
  }
}

// clip job row: {on}; x <- min(max(x, cf min x), cf max x)
__global__ void __launch_bounds__(RED_THREADS)
clip_kernel(float* x, long ldx, const long* __restrict__ jobs, const double* __restrict__ cf, int T) {
  pdl_wait();
  __shared__ float smn[32], smx[32];
  const int b = blockIdx.x;
  if (jobs[b] == 0) return;
  float* xr = x + (long)b * ldx;
  float mn = INFINITY, mx = -INFINITY;
  for (long t = threadIdx.x; t < T; t += blockDim.x) {
    mn = fminf(mn, xr[t]);
    mx = fmaxf(mx, xr[t]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { smn[w] = mn; smx[w] = mx; }
  __syncthreads();
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { mn = fminf(mn, smn[i]); mx = fmaxf(mx, smx[i]); }
  const float lo = (float)(cf[b] * (double)mn), hi = (float)(cf[b] * (double)mx);
  for (long t = threadIdx.x; t < T; t += blockDim.x) xr[t] = fminf(fmaxf(xr[t], lo), hi);
}

// label[b, j] = mean over [j*d, (j+1)*d) of (t >= shift), 0 for samples without overlap
__global__ void overlap_label_kernel(const long* __restrict__ jobs, int T, int d,
                                     float* __restrict__ label, long ldl) {
  pdl_wait();
  const int b = blockIdx.y, nl = T / d;
  const long* r = jobs + (long)b * 3;
  const bool on = r[0] != 0 && r[1] >= 0 && r[1] < T;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nl; j += gridDim.x * blockDim.x) {
    float v = 0.f;
    if (on) {
      const long lo = max((long)j * d, r[1]), hi = (long)(j + 1) * d;
      v = (float)(hi > lo ? hi - lo : 0) / (float)d;
    }
    label[(long)b * ldl + j] = v;
  }
}

int set_smem(const void* fn, size_t bytes, const char* who) {
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    pase_set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e));
    return (int)e;
  }
  return PASE_OK;
}

constexpr int MAX_T = 1 << 24;
constexpr int MAX_L = 1 << 20;
constexpr int MAX_JOBS = 65535;

int conv_geometry(int njobs, int T, int Lmax, int* nbmax, int* pmax, long* bytes) {
  PASE_CHECK_ARG(njobs > 0 && njobs <= MAX_JOBS, "pase_fft_conv: njobs=%d outside [1, %d]", njobs, MAX_JOBS);
  PASE_CHECK_ARG(T > 0 && T <= MAX_T, "pase_fft_conv: T=%d outside [1, %d]", T, MAX_T);
  PASE_CHECK_ARG(Lmax > 0 && Lmax <= MAX_L, "pase_fft_conv: Lmax=%d outside [1, %d]", Lmax, MAX_L);
  *nbmax = (int)(((long)T + Lmax - 1 + BLK - 1) / BLK);
  *pmax = (Lmax + BLK - 1) / BLK;
  // spectra (X then H), energy partials, the unscaled window
  *bytes = (long)njobs * (*nbmax + *pmax) * FFT_N * (long)sizeof(float2) +
           (long)njobs * *nbmax * (long)sizeof(double) + (long)njobs * T * (long)sizeof(float);
  return PASE_OK;
}

}  // namespace

extern "C" {

int pase_fft_conv_workspace(int njobs, int T, int Lmax, long* bytes) {
  PASE_CHECK_ARG(bytes, "pase_fft_conv_workspace: bytes is NULL");
  int nb, pm;
  return conv_geometry(njobs, T, Lmax, &nb, &pm, bytes);
}

int pase_fft_conv(const float* x, long ldx, const float* bank, long bank_len, const long* jobs,
                  int njobs, int T, int Lmax, const float* twiddle, void* ws, long ws_bytes,
                  float* out, long ldo, void* stream) {
  int nbmax, pmax;
  long need;
  int rc = conv_geometry(njobs, T, Lmax, &nbmax, &pmax, &need);
  if (rc != PASE_OK) return rc;
  PASE_CHECK_ARG(x, "pase_fft_conv: x is NULL");
  PASE_CHECK_ARG(bank, "pase_fft_conv: bank is NULL");
  PASE_CHECK_ARG(jobs, "pase_fft_conv: jobs is NULL");
  PASE_CHECK_ARG(twiddle, "pase_fft_conv: twiddle is NULL");
  PASE_CHECK_ARG(ws, "pase_fft_conv: ws is NULL");
  PASE_CHECK_ARG(out, "pase_fft_conv: out is NULL");
  PASE_CHECK_ARG(bank_len > 0, "pase_fft_conv: bank_len=%ld", bank_len);
  PASE_CHECK_ARG(ldx >= T, "pase_fft_conv: ldx=%ld < T=%d", ldx, T);
  PASE_CHECK_ARG(ldo >= T, "pase_fft_conv: ldo=%ld < T=%d", ldo, T);
  PASE_CHECK_ARG(ws_bytes >= need, "pase_fft_conv: ws_bytes=%ld < %ld", ws_bytes, need);
  PASE_CHECK_ARG(aligned16(ws), "pase_fft_conv: ws is not 16-byte aligned");
  PASE_CHECK_ARG((reinterpret_cast<uintptr_t>(twiddle) & 7u) == 0, "pase_fft_conv: twiddle is not 8-byte aligned");
  static bool smem_set = false;
  if (!smem_set) {
    if ((rc = set_smem((const void*)conv_spectra_kernel, FFT_SMEM, "pase_fft_conv")) != PASE_OK) return rc;
    if ((rc = set_smem((const void*)conv_output_kernel, FFT_SMEM, "pase_fft_conv")) != PASE_OK) return rc;
    smem_set = true;
  }
  float2* xspec = reinterpret_cast<float2*>(ws);
  float2* hspec = xspec + (long)njobs * nbmax * FFT_N;
  double* epart = reinterpret_cast<double*>(hspec + (long)njobs * pmax * FFT_N);
  float* y = reinterpret_cast<float*>(epart + (long)njobs * nbmax);
  const float2* tw = reinterpret_cast<const float2*>(twiddle);
  cudaStream_t st = (cudaStream_t)stream;
  PASE_LAUNCH((conv_spectra_kernel), dim3(nbmax + pmax, njobs), FFT_THREADS, FFT_SMEM, st, x, ldx,
              bank, bank_len, jobs, T, Lmax, nbmax, pmax, tw, xspec, hspec);
  PASE_LAUNCH_CHECK("pase_fft_conv(spectra)");
  PASE_LAUNCH((conv_output_kernel), dim3(nbmax, njobs), FFT_THREADS, FFT_SMEM, st, jobs, T, Lmax,
              bank_len, nbmax, pmax, tw, (const float2*)xspec, (const float2*)hspec, y, epart);
  PASE_LAUNCH_CHECK("pase_fft_conv(output)");
  PASE_LAUNCH((conv_scale_kernel), dim3(njobs), RED_THREADS, 0, st, x, ldx, jobs, T, Lmax,
              bank_len, nbmax, (const float*)y, (const double*)epart, out, ldo);
  PASE_LAUNCH_CHECK("pase_fft_conv(scale)");
  return PASE_OK;
}

int pase_segment_gather(const float* pool, long pool_len, const long* jobs, int njobs, int T,
                        float* out, long ldo, void* stream) {
  PASE_CHECK_ARG(pool, "pase_segment_gather: pool is NULL");
  PASE_CHECK_ARG(jobs, "pase_segment_gather: jobs is NULL");
  PASE_CHECK_ARG(out, "pase_segment_gather: out is NULL");
  PASE_CHECK_ARG(pool_len > 0, "pase_segment_gather: pool_len=%ld", pool_len);
  PASE_CHECK_ARG(njobs > 0 && njobs <= MAX_JOBS, "pase_segment_gather: njobs=%d outside [1, %d]", njobs, MAX_JOBS);
  PASE_CHECK_ARG(T > 0 && T <= MAX_T, "pase_segment_gather: T=%d outside [1, %d]", T, MAX_T);
  PASE_CHECK_ARG(ldo >= T, "pase_segment_gather: ldo=%ld < T=%d", ldo, T);
  const int bx = (int)std::min<long>(((long)T + 255) / 256, 64);
  PASE_LAUNCH((segment_gather_kernel), dim3(bx, njobs), 256, 0, (cudaStream_t)stream, pool,
              pool_len, jobs, T, out, ldo);
  PASE_LAUNCH_CHECK("pase_segment_gather");
  return PASE_OK;
}

int pase_noise_mix(float* x, long ldx, const float* seg, long lds, const long* jobs,
                   const double* snr_lin, int njobs, int T, void* stream) {
  PASE_CHECK_ARG(x, "pase_noise_mix: x is NULL");
  PASE_CHECK_ARG(seg, "pase_noise_mix: seg is NULL");
  PASE_CHECK_ARG(jobs, "pase_noise_mix: jobs is NULL");
  PASE_CHECK_ARG(snr_lin, "pase_noise_mix: snr_lin is NULL");
  PASE_CHECK_ARG(njobs > 0 && njobs <= MAX_JOBS, "pase_noise_mix: njobs=%d outside [1, %d]", njobs, MAX_JOBS);
  PASE_CHECK_ARG(T > 0 && T <= MAX_T, "pase_noise_mix: T=%d outside [1, %d]", T, MAX_T);
  PASE_CHECK_ARG(ldx >= T, "pase_noise_mix: ldx=%ld < T=%d", ldx, T);
  PASE_CHECK_ARG(lds >= T, "pase_noise_mix: lds=%ld < T=%d", lds, T);
  PASE_LAUNCH((noise_mix_kernel), dim3(njobs), RED_THREADS, 0, (cudaStream_t)stream, x, ldx, seg,
              lds, jobs, snr_lin, T);
  PASE_LAUNCH_CHECK("pase_noise_mix");
  return PASE_OK;
}

int pase_clip(float* x, long ldx, const long* jobs, const double* cf, int njobs, int T, void* stream) {
  PASE_CHECK_ARG(x, "pase_clip: x is NULL");
  PASE_CHECK_ARG(jobs, "pase_clip: jobs is NULL");
  PASE_CHECK_ARG(cf, "pase_clip: cf is NULL");
  PASE_CHECK_ARG(njobs > 0 && njobs <= MAX_JOBS, "pase_clip: njobs=%d outside [1, %d]", njobs, MAX_JOBS);
  PASE_CHECK_ARG(T > 0 && T <= MAX_T, "pase_clip: T=%d outside [1, %d]", T, MAX_T);
  PASE_CHECK_ARG(ldx >= T, "pase_clip: ldx=%ld < T=%d", ldx, T);
  PASE_LAUNCH((clip_kernel), dim3(njobs), RED_THREADS, 0, (cudaStream_t)stream, x, ldx, jobs, cf, T);
  PASE_LAUNCH_CHECK("pase_clip");
  return PASE_OK;
}

int pase_overlap_label(const long* jobs, int njobs, int T, int d, float* label, long ldl,
                       void* stream) {
  PASE_CHECK_ARG(jobs, "pase_overlap_label: jobs is NULL");
  PASE_CHECK_ARG(label, "pase_overlap_label: label is NULL");
  PASE_CHECK_ARG(njobs > 0 && njobs <= MAX_JOBS, "pase_overlap_label: njobs=%d outside [1, %d]", njobs, MAX_JOBS);
  PASE_CHECK_ARG(T > 0 && T <= MAX_T, "pase_overlap_label: T=%d outside [1, %d]", T, MAX_T);
  PASE_CHECK_ARG(d > 0 && T % d == 0, "pase_overlap_label: d=%d does not divide T=%d", d, T);
  PASE_CHECK_ARG(ldl >= T / d, "pase_overlap_label: ldl=%ld < T/d=%d", ldl, T / d);
  const int nl = T / d;
  const int bx = std::min((nl + 255) / 256, 64);
  PASE_LAUNCH((overlap_label_kernel), dim3(bx, njobs), 256, 0, (cudaStream_t)stream, jobs, T, d,
              label, ldl);
  PASE_LAUNCH_CHECK("pase_overlap_label");
  return PASE_OK;
}

}  // extern "C"
