// Sample history of a StreamPool (pase_b200/frontend.py): one ring of ring_cap samples per
// stream slot in a device arena, and the round's packed waveform gathered from it.
//
//   pase_stream_gather   per table row {slot, head, nnew, stage_off, ring_s, old, seg_len,
//                        wave_off}: appends the stream's nnew new samples staging[stage_off..]
//                        at ring position head (mod ring_cap), and writes its segment's seg_len
//                        samples to wave[wave_off..]: the first `old` from the ring from position
//                        ring_s, the rest from staging (old may be negative: the segment then
//                        starts -old samples into this round's new ones).
//
// The host (StreamPool) sizes a ring so that the samples a segment reads from it and the ones
// appended in the same launch never share a position (ring_cap >= samples kept + one piece), so
// the two halves of a row need no ordering.
#include "common.cuh"

namespace {

constexpr int GATHER_THREADS = 256;
constexpr int GATHER_ITEMS = 4;                 // samples per thread and block-row pass

__global__ void __launch_bounds__(GATHER_THREADS)
stream_gather_kernel(const float* __restrict__ staging, float* __restrict__ ring, long ring_cap,
                     float* __restrict__ wave, const int* __restrict__ tab) {
  pdl_wait();
  const int* row = tab + 8 * blockIdx.y;
  const long slot = __ldg(row), head = __ldg(row + 1);
  const int nnew = __ldg(row + 2);
  const long stage_off = __ldg(row + 3), ring_s = __ldg(row + 4);
  const int old = __ldg(row + 5), seg_len = __ldg(row + 6);
  const long wave_off = __ldg(row + 7);
  float* r = ring + slot * ring_cap;            // 64-bit arena offset
  const float* st = staging + stage_off;
  const int n = max(nnew, seg_len);
  for (int i = blockIdx.x * GATHER_THREADS + threadIdx.x; i < n;
       i += gridDim.x * GATHER_THREADS) {
    if (i < nnew) {
      long p = head + i;
      if (p >= ring_cap) p -= ring_cap;
      r[p] = st[i];
    }
    if (i < seg_len) {
      float v;
      if (i < old) {
        long p = ring_s + i;
        if (p >= ring_cap) p -= ring_cap;
        v = r[p];
      } else {
        v = st[i - old];
      }
      wave[wave_off + i] = v;
    }
  }
}

}  // namespace

int pase_stream_gather(const float* staging, float* ring, long ring_cap, float* wave,
                       const int* tab, int nrow, int max_len, void* stream) {
  PASE_CHECK_ARG(ring && wave && tab, "pase_stream_gather: null pointer");
  PASE_CHECK_ARG(nrow > 0 && nrow <= 65535 && max_len >= 0 && ring_cap > 0,
                 "pase_stream_gather: nrow=%d max_len=%d ring_cap=%ld", nrow, max_len, ring_cap);
  PASE_CHECK_ARG(max_len <= ring_cap, "pase_stream_gather: max_len=%d past ring_cap=%ld",
                 max_len, ring_cap);
  const int per = GATHER_THREADS * GATHER_ITEMS;
  const int bx = max(1, (max_len + per - 1) / per);
  PASE_LAUNCH((stream_gather_kernel), dim3(bx, nrow), GATHER_THREADS, 0, (cudaStream_t)stream,
              staging, ring, ring_cap, wave, tab);
  PASE_LAUNCH_CHECK("pase_stream_gather");
  return PASE_OK;
}
