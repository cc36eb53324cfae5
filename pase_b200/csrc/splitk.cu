// Split-K weight gradients (pase_tc_gemm_tn, pase_gemm_tn): the shared partial-tile workspace
// and the reduction that sums the splits in split order, so that the result does not depend
// on the order in which the splits finish.
#include "common.cuh"

namespace {

constexpr int SK_BM = 128;      // tile rows of both weight-gradient kernels

// C[i, j] (+)= sum over the splits, in split order, of the partial tiles holding (i, j)
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, int splits, int tiles_j, int bn,
                                     long tiles, float* __restrict__ C, long ldc, int I, int J,
                                     int accumulate) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)I * J) return;
  const int i = (int)(idx / J), j = (int)(idx % J);
  const long tile_elems = (long)SK_BM * bn;
  const float* p = ws + ((long)(i / SK_BM) * tiles_j + j / bn) * tile_elems + (i % SK_BM) * bn + j % bn;
  float sum = 0.f;
  for (int z = 0; z < splits; ++z) sum += p[z * tiles * tile_elems];
  float* c = C + (long)i * ldc + j;
  *c = accumulate ? *c + sum : sum;
}

}  // namespace

long pase_splitk_ws_tiles() { return (long)PASE_SPLITK_WAVES * pase_num_sms(); }

// allocated once per device on first use, never freed: captured CUDA graphs keep using it
float* pase_splitk_workspace(cudaStream_t st, const char* who) {
  static float* ws[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) {
    pase_set_error("%s: device index %d", who, dev);
    return nullptr;
  }
  if (ws[dev] != nullptr) return ws[dev];
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  if (cs != cudaStreamCaptureStatusNone) {
    pase_set_error("%s: first split-K call on this device inside a stream capture "
                   "(run one step before capturing)", who);
    return nullptr;
  }
  cudaError_t e = cudaMalloc(&ws[dev], (size_t)pase_splitk_ws_tiles() * PASE_SPLITK_TILE *
                                           sizeof(float));
  if (e != cudaSuccess) {
    ws[dev] = nullptr;
    pase_set_error("%s: workspace allocation: %s", who, cudaGetErrorString(e));
    return nullptr;
  }
  return ws[dev];
}

int pase_splitk_reduce(const float* ws, int splits, int tiles_j, int bn, long tiles, float* C,
                       long ldc, int I, int J, int accumulate, cudaStream_t st, const char* who) {
  const long n = (long)I * J;
  splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws, splits, tiles_j, bn, tiles,
                                                                   C, ldc, I, J, accumulate);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    pase_set_error("%s (split reduction): launch failed: %s", who, cudaGetErrorString(e));
    return (int)e;
  }
  return PASE_OK;
}
