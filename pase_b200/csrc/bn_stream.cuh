// Internal interface between act.cu (C-ABI entry points, register-resident kernels) and
// bn_stream.cu (bulk-copy staged persistent kernels for the BatchNorm/PReLU backward passes).
#pragma once
#include "common.cuh"

// gradient sources of one encoder block's output (see pase_bn_prelu_bwd_reduce)
struct BwdSrc {
  const void* A; long a_ss, a_rs; int padL, padR;
  const float* B; long b_ss, b_rs; int b_shift;
  const float* P; long p_ss, p_rs; int pool_d, pool_T;
};

struct BnStreamArgs {
  const void* y; int y_bf16; long y_ss; int N, T, C;
  const float *mean, *invstd, *gamma, *scale, *shift, *alpha;
  BwdSrc s; int a_bf16;
  // pass 1 (sums)
  double *S1, *S2, *dalpha; float* amax;
  // pass 2 (dy)
  const double *S1in, *S2in; double inv_count;
  void *dst, *dst_lo; int dst_fmt; long d_ss; double* dbias; float* scale_out;
};

// how the staged kernels cut a call: tiles of TT = 4096 / C time steps, tps tiles per sample,
// total = N * tps tiles, shared by grid persistent blocks
struct BnStreamPlan { int TT, tps; long total, grid; };

// true when the staged kernels support the shape / alignment (else: register kernels)
bool pase_bn_stream_ok(const BnStreamArgs& a);
BnStreamPlan pase_bn_stream_plan(const BnStreamArgs& a);
int pase_bn_stream_reduce(const BnStreamArgs& a, cudaStream_t st);
int pase_bn_stream_apply(const BnStreamArgs& a, cudaStream_t st);
