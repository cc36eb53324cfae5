// On-device BATCH ASSEMBLY (DESIGN.md section 12, row f-N2): the per-sample work of the
// reference's DataLoader -- the chunk windows of SingleChunkWav / MIChunkWav
// (pase/transforms.py:295-436) with their reflect padding and norm_and_scale, and the frame
// slices CachedCompose takes from precomputed features (transforms.py:253-292) -- as two gathers
// from a corpus resident in HBM or in mapped page-locked host memory.  The host planner
// (pase_b200/batch.py) draws the windows and validates every row, so launch shapes depend only
// on (B, sources, T, F, frames) and one uploaded table plus these launches can be captured in a
// CUDA graph.
//
//   pase_chunk_gather   one CTA per (source, sample): max|x| over the window, then the scaled
//                       window (and the clean copy cchunk of the first source)
//   pase_frames_gather  out[b, f, t] = pool[off_b + f * frames_b + s_b + t], coalesced along t
#include <algorithm>
#include "common.cuh"

namespace {

constexpr int CHUNK_THREADS = 512;
constexpr int CR = 6;                 // chunk row: {fmt, off, L, beg, scale, rbits}
constexpr int FR = 3;                 // frames row: {off, frames, s}
constexpr float PCM_SCALE = 1.f / 32768.f;

struct ChunkRow {
  long off, L, beg;
  int fmt;
  bool scale, on;
  float r;
};

__device__ __forceinline__ ChunkRow load_chunk_row(const long* rows, long pcm_len, long flt_len, int T) {
  ChunkRow c;
  c.fmt = (int)rows[0]; c.off = rows[1]; c.L = rows[2]; c.beg = rows[3];
  c.scale = rows[4] != 0;
  c.r = __int_as_float((int)rows[5]);
  const long len = c.fmt == 0 ? pcm_len : flt_len;
  // window in range, or reflect padding by P = T - L < L from beg = 0 (F.pad's limit)
  const bool win = c.L >= 1 && c.beg >= 0 &&
                   (c.beg + T <= c.L || (c.beg == 0 && (long)T - c.L < c.L));
  c.on = (c.fmt == 0 || c.fmt == 1) && c.off >= 0 && c.off + c.L <= len && win;
  return c;
}

__device__ __forceinline__ float chunk_at(const short* __restrict__ pcm, const float* __restrict__ flt,
                                          const ChunkRow& c, long j) {
  long p = c.beg + j;
  if (p >= c.L) p = 2 * c.L - 2 - p;                // reflect: u[L + i] = u[L - 2 - i]
  return c.fmt == 0 ? (float)pcm[c.off + p] * PCM_SCALE : flt[c.off + p];
}

__global__ void __launch_bounds__(CHUNK_THREADS)
chunk_gather_kernel(const short* __restrict__ pcm, long pcm_len, const float* __restrict__ flt,
                    long flt_len, const long* __restrict__ rows, int nsrc, int T, int cchunk,
                    float* __restrict__ out, long plane) {
  pdl_wait();
  __shared__ float red[CHUNK_THREADS / 32];
  const int s = blockIdx.x, b = blockIdx.y;
  const ChunkRow c = load_chunk_row(rows + ((long)b * nsrc + s) * CR, pcm_len, flt_len, T);
  if (!c.on) return;
  float m = 0.f;
  if (c.scale) {
    // max|x| is exact in any order; fmaxf keeps the first operand that is not NaN
    for (long j = threadIdx.x; j < T; j += blockDim.x) m = fmaxf(m, fabsf(chunk_at(pcm, flt, c, j)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
  }
  float* o = out + (long)s * plane + (long)b * T;
  float* o2 = (s == 0 && cchunk) ? out + (long)nsrc * plane + (long)b * T : nullptr;
  for (long j = threadIdx.x; j < T; j += blockDim.x) {
    float v = chunk_at(pcm, flt, c, j);
    // torch's CPU `wav / max(abs(wav)) * rand`: two correctly rounded fp32 operations
    if (c.scale) v = __fmul_rn(__fdiv_rn(v, m), c.r);
    o[j] = v;
    if (o2) o2[j] = v;
  }
}

__global__ void frames_gather_kernel(const float* __restrict__ pool, long pool_len,
                                     const long* __restrict__ rows, int F, int n,
                                     float* __restrict__ out) {
  pdl_wait();
  const int b = blockIdx.y;
  const long* r = rows + (long)b * FR;
  const long off = r[0], frames = r[1], s = r[2];
  if (off < 0 || s < 0 || s + n > frames || off + (long)F * frames > pool_len) return;
  const long total = (long)F * n;
  float* o = out + (long)b * total;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const long f = i / n, t = i - f * n;
    o[i] = pool[off + f * frames + s + t];
  }
}

constexpr int MAX_T = 1 << 24;
constexpr int MAX_B = 65535;

}  // namespace

extern "C" {

int pase_chunk_gather(const void* pcm, long pcm_len, const float* flt, long flt_len,
                      const long* rows, int B, int nsrc, int T, int cchunk, float* out,
                      long plane, void* stream) {
  PASE_CHECK_ARG(pcm || flt, "pase_chunk_gather: both pools are NULL");
  PASE_CHECK_ARG(pcm_len >= 0 && (pcm || pcm_len == 0), "pase_chunk_gather: pcm_len=%ld", pcm_len);
  PASE_CHECK_ARG(flt_len >= 0 && (flt || flt_len == 0), "pase_chunk_gather: flt_len=%ld", flt_len);
  PASE_CHECK_ARG(rows, "pase_chunk_gather: rows is NULL");
  PASE_CHECK_ARG(out, "pase_chunk_gather: out is NULL");
  PASE_CHECK_ARG(B > 0 && B <= MAX_B, "pase_chunk_gather: B=%d outside [1, %d]", B, MAX_B);
  PASE_CHECK_ARG(nsrc >= 1 && nsrc <= 3, "pase_chunk_gather: nsrc=%d outside [1, 3]", nsrc);
  PASE_CHECK_ARG(T > 0 && T <= MAX_T, "pase_chunk_gather: T=%d outside [1, %d]", T, MAX_T);
  PASE_CHECK_ARG(plane >= (long)B * T, "pase_chunk_gather: plane=%ld < B*T=%ld", plane, (long)B * T);
  PASE_LAUNCH((chunk_gather_kernel), dim3(nsrc, B), CHUNK_THREADS, 0, (cudaStream_t)stream,
              (const short*)pcm, pcm_len, flt, flt_len, rows, nsrc, T, cchunk, out, plane);
  PASE_LAUNCH_CHECK("pase_chunk_gather");
  return PASE_OK;
}

int pase_frames_gather(const float* pool, long pool_len, const long* rows, int B, int F, int n,
                       float* out, void* stream) {
  PASE_CHECK_ARG(pool, "pase_frames_gather: pool is NULL");
  PASE_CHECK_ARG(pool_len > 0, "pase_frames_gather: pool_len=%ld", pool_len);
  PASE_CHECK_ARG(rows, "pase_frames_gather: rows is NULL");
  PASE_CHECK_ARG(out, "pase_frames_gather: out is NULL");
  PASE_CHECK_ARG(B > 0 && B <= MAX_B, "pase_frames_gather: B=%d outside [1, %d]", B, MAX_B);
  PASE_CHECK_ARG(F > 0 && n > 0 && (long)F * n <= MAX_T, "pase_frames_gather: F=%d n=%d", F, n);
  const long total = (long)F * n;
  const int bx = (int)std::min<long>((total + 255) / 256, 64);
  PASE_LAUNCH((frames_gather_kernel), dim3(bx, B), 256, 0, (cudaStream_t)stream, pool, pool_len,
              rows, F, n, out);
  PASE_LAUNCH_CHECK("pase_frames_gather");
  return PASE_OK;
}

}  // extern "C"
