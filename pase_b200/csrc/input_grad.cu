// Input gradient of the sinc layer (the waveform gradient of WaveFe): the transposed band-pass
// convolution runs as one polyphase NT GEMM on the existing kernels (DESIGN.md section 17); the
// kernels here prepare its operands and fold the reflect pad back.
//
//   pase_sinc_dgrad_pack    dy (N samples x src_frames frames x C channels, operand format)
//                           -> the GEMM's A operand: per sample dst_frames frames, frame e holding
//                           dy frame e - halo, zero outside [0, T_out).  Byte copy, so every
//                           operand format (and its lo twin) passes through unchanged.
//   pase_sinc_dgrad_weight  band-pass bank filt (C x k) -> the banded B operand
//                           Wdg[p, (r, q, co)] = filt[co][H + p - fold r - q] (0 outside [0, k)).
//   pase_reflect_fold_wave  d(reflect-padded rows) -> d(waveform): the adjoint of
//                           pase_reflect_pad_wave, one gather per output sample.
#include "common.cuh"

namespace {

constexpr int THREADS = 256;

// U: the copy unit (uint4 when a frame's bytes are a multiple of 16, else uint2)
template <typename U>
__global__ void __launch_bounds__(THREADS)
sinc_dgrad_pack_kernel(const U* __restrict__ src, const U* __restrict__ src_lo, U* __restrict__ dst,
                       U* __restrict__ dst_lo, int units, int T_out, long src_frames, int halo,
                       long dst_frames, long total) {
  pdl_wait();
  for (long i = (long)blockIdx.x * THREADS + threadIdx.x; i < total;
       i += (long)gridDim.x * THREADS) {
    const long fr = i / units;
    const int c = (int)(i - fr * units);
    const long n = fr / dst_frames;
    const long t = fr - n * dst_frames - halo;
    U v = {}, w = {};
    if (t >= 0 && t < T_out) {
      const long o = (n * src_frames + t) * units + c;
      v = src[o];
      if (dst_lo != nullptr) w = src_lo[o];
    }
    dst[i] = v;
    if (dst_lo != nullptr) dst_lo[i] = w;
  }
}

__global__ void __launch_bounds__(THREADS)
sinc_dgrad_weight_kernel(const float* __restrict__ filt, float* __restrict__ Wdg, int C, int k,
                         int fold, int rows, long total) {
  pdl_wait();
  const int H = (rows - 1) * fold;
  const long Kd = (long)rows * fold * C;
  for (long i = (long)blockIdx.x * THREADS + threadIdx.x; i < total;
       i += (long)gridDim.x * THREADS) {
    const int p = (int)(i / Kd);
    const int kk = (int)(i - p * Kd);
    const int rq = kk / C, co = kk - rq * C;       // rq = fold r + q
    const int j = H + p - rq;
    Wdg[i] = (j >= 0 && j < k) ? __ldg(filt + (long)co * k + j) : 0.f;
  }
}

// One utterance's fold: o[t] = (+= when ACC) its padded-waveform gradient at t, plus the mirrored
// pad gradient on the sides where the pad reflects the utterance itself (fold_l / fold_r)
template <bool ACC>
__device__ __forceinline__ void reflect_fold_wave_utt(const float* __restrict__ d,
                                                      float* __restrict__ o, int T, int padL,
                                                      int padR, bool fold_l, bool fold_r) {
  for (int t = blockIdx.x * THREADS + threadIdx.x; t < T; t += gridDim.x * THREADS) {
    float v = d[t + padL];
    if (fold_l && t >= 1 && t <= padL) v += d[padL - t];                           // left mirror
    if (fold_r && t >= T - 1 - padR && t <= T - 2) v += d[padL + 2 * (T - 1) - t]; // right mirror
    if constexpr (ACC) o[t] += v;
    else o[t] = v;
  }
}

__global__ void __launch_bounds__(THREADS)
reflect_fold_wave_kernel(const float* __restrict__ dpad, long pitch, float* __restrict__ dx, int T,
                         int padL, int padR) {
  pdl_wait();
  const int n = blockIdx.y;
  reflect_fold_wave_utt<false>(dpad + (long)n * pitch, dx + (long)n * T, T, padL, padR, true,
                               true);
}

// pase_reflect_fold_wave for utterance blockIdx.y of a packed waveform: tab row {x_off, T, dst_off}
__global__ void __launch_bounds__(THREADS)
reflect_fold_wave_var_kernel(const float* __restrict__ dpad, const int* __restrict__ tab,
                             float* __restrict__ dx, int padL, int padR) {
  pdl_wait();
  const int* r = tab + 3 * blockIdx.y;
  reflect_fold_wave_utt<false>(dpad + __ldg(r + 2), dx + __ldg(r), __ldg(r + 1), padL, padR, true,
                               true);
}

// One window of a recording (WaveFe.encode_long): dx[x0 + t] += the window's padded-waveform
// gradient at t, folding the pad only on the sides where the window's pad is the recording's own
__global__ void __launch_bounds__(THREADS)
reflect_fold_wave_acc_kernel(const float* __restrict__ d, float* __restrict__ dx, long x0, int T,
                             int padL, int padR, int fold_l, int fold_r) {
  pdl_wait();
  reflect_fold_wave_utt<true>(d, dx + x0, T, padL, padR, fold_l, fold_r);
}

inline unsigned grid_for(long total) {
  long b = (total + THREADS - 1) / THREADS;
  const long cap = (long)pase_num_sms() * 16;
  return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

int pase_sinc_dgrad_pack(const void* src, const void* src_lo, void* dst, void* dst_lo, int esz,
                         int N, int C, int T_out, long src_frames, int halo, long dst_frames,
                         void* stream) {
  PASE_CHECK_ARG(src && dst && (src_lo == nullptr) == (dst_lo == nullptr),
                 "pase_sinc_dgrad_pack: null pointer / lo pair");
  PASE_CHECK_ARG((esz == 2 || esz == 4) && N > 0 && C > 0 && (C * esz) % 8 == 0 && T_out > 0 &&
                     src_frames >= T_out && halo >= 0 && dst_frames >= halo + T_out,
                 "pase_sinc_dgrad_pack: bad shape (esz=%d N=%d C=%d T_out=%d src_frames=%ld "
                 "halo=%d dst_frames=%ld)", esz, N, C, T_out, src_frames, halo, dst_frames);
  cudaStream_t st = (cudaStream_t)stream;
  const bool wide = (C * esz) % 16 == 0 && aligned16(src) && aligned16(dst) &&
                    (src_lo == nullptr || (aligned16(src_lo) && aligned16(dst_lo)));
  if (wide) {
    const int units = C * esz / 16;
    const long total = (long)N * dst_frames * units;
    PASE_LAUNCH((sinc_dgrad_pack_kernel<uint4>), grid_for(total), THREADS, 0, st,
                (const uint4*)src, (const uint4*)src_lo, (uint4*)dst, (uint4*)dst_lo, units, T_out,
                src_frames, halo, dst_frames, total);
  } else {
    PASE_CHECK_ARG(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 7u) == 0,
                   "pase_sinc_dgrad_pack: operands must be 8-byte aligned");
    const int units = C * esz / 8;
    const long total = (long)N * dst_frames * units;
    PASE_LAUNCH((sinc_dgrad_pack_kernel<uint2>), grid_for(total), THREADS, 0, st,
                (const uint2*)src, (const uint2*)src_lo, (uint2*)dst, (uint2*)dst_lo, units, T_out,
                src_frames, halo, dst_frames, total);
  }
  PASE_LAUNCH_CHECK("pase_sinc_dgrad_pack");
  return PASE_OK;
}

int pase_sinc_dgrad_weight(const float* filt, float* Wdg, int C, int k, int fold, int rows,
                           void* stream) {
  PASE_CHECK_ARG(filt && Wdg, "pase_sinc_dgrad_weight: null pointer");
  PASE_CHECK_ARG(C > 0 && k > 0 && fold > 0 && rows >= 1 && (rows - 1) * fold >= k - 1,
                 "pase_sinc_dgrad_weight: rows=%d fold=%d do not span k=%d taps", rows, fold, k);
  const long total = (long)fold * rows * fold * C;
  PASE_LAUNCH((sinc_dgrad_weight_kernel), grid_for(total), THREADS, 0, (cudaStream_t)stream, filt,
              Wdg, C, k, fold, rows, total);
  PASE_LAUNCH_CHECK("pase_sinc_dgrad_weight");
  return PASE_OK;
}

int pase_reflect_fold_wave(const float* dpad, long pitch, float* dx, int N, int T, int padL,
                           int padR, void* stream) {
  PASE_CHECK_ARG(dpad && dx && N > 0 && T > 0 && padL >= 0 && padR >= 0,
                 "pase_reflect_fold_wave: bad args");
  PASE_CHECK_ARG(padL < T && padR < T, "pase_reflect_fold_wave: reflect pad (%d,%d) >= T=%d", padL,
                 padR, T);
  PASE_CHECK_ARG(pitch >= (long)T + padL + padR,
                 "pase_reflect_fold_wave: pitch %ld < padded length %d", pitch, T + padL + padR);
  dim3 grid((unsigned)((T + THREADS - 1) / THREADS), N);
  PASE_LAUNCH((reflect_fold_wave_kernel), grid, THREADS, 0, (cudaStream_t)stream, dpad, pitch, dx,
              T, padL, padR);
  PASE_LAUNCH_CHECK("pase_reflect_fold_wave");
  return PASE_OK;
}

int pase_reflect_fold_wave_var(const float* dpad, const int* tab, int nseg, int max_T, float* dx,
                               int padL, int padR, void* stream) {
  PASE_CHECK_ARG(dpad && tab && dx && nseg > 0 && nseg <= 65535 && max_T > 0 && padL >= 0 &&
                     padR >= 0, "pase_reflect_fold_wave_var: bad args");
  dim3 grid((unsigned)((max_T + THREADS - 1) / THREADS), nseg);
  PASE_LAUNCH((reflect_fold_wave_var_kernel), grid, THREADS, 0, (cudaStream_t)stream, dpad, tab,
              dx, padL, padR);
  PASE_LAUNCH_CHECK("pase_reflect_fold_wave_var");
  return PASE_OK;
}

int pase_reflect_fold_wave_acc(const float* dpad, float* dx, long x0, int T, int padL, int padR,
                               int fold_l, int fold_r, void* stream) {
  PASE_CHECK_ARG(dpad && dx && x0 >= 0 && T > 0 && padL >= 0 && padR >= 0 && padL < T &&
                     padR < T, "pase_reflect_fold_wave_acc: bad args (x0=%ld T=%d pad %d,%d)", x0,
                 T, padL, padR);
  PASE_LAUNCH((reflect_fold_wave_acc_kernel), dim3((unsigned)((T + THREADS - 1) / THREADS)),
              THREADS, 0, (cudaStream_t)stream, dpad, dx, x0, T, padL, padR, fold_l, fold_r);
  PASE_LAUNCH_CHECK("pase_reflect_fold_wave_acc");
  return PASE_OK;
}
