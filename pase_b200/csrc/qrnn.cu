// QRNN (window=2) gate activations + ForgetMult recurrence + output gate, forward and
// backward.  One thread per (sample, hidden unit); time is sequential (T' = T/160
// frames), loads are issued UNROLL steps ahead of the dependent recurrence.
// Replaces torchqrnn's runtime-compiled recurrent_forget_mult kernels
// (reference call site: pase/models/modules.py:52, frontend.py:256-259).
#include "common.cuh"

namespace {

constexpr int UNROLL = 8;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// One sample's sequential scan of hidden unit c: y / hp / cp point at its first time step,
// cprev is the cell state before it (0 at the start of an utterance).  Returns the state after
// the last step.  Every step runs the same arithmetic whether it falls in an unrolled group or
// in the remainder, so a scan cut into pieces that carry the state reproduces the whole scan's
// bits (pase_qrnn_scan_fwd_carry_var).
__device__ __forceinline__ float qrnn_fwd_seq(const float* __restrict__ y, float* __restrict__ hp,
                                              long ldh, float* __restrict__ cp, int T, int H,
                                              float cprev) {
  int t = 0;
  for (; t + UNROLL <= T; t += UNROLL) {
    float z[UNROLL], f[UNROLL], o[UNROLL];
#pragma unroll
    for (int i = 0; i < UNROLL; ++i) {
      const float* yr = y + (long)(t + i) * 3 * H;
      z[i] = yr[0]; f[i] = yr[H]; o[i] = yr[2 * H];
    }
#pragma unroll
    for (int i = 0; i < UNROLL; ++i) {
      const float zz = tanhf(z[i]), ff = sigmoidf_(f[i]), oo = sigmoidf_(o[i]);
      cprev = ff * zz + (1.f - ff) * cprev;
      cp[(long)(t + i) * H] = cprev;
      hp[(long)(t + i) * ldh] = oo * cprev;
    }
  }
  for (; t < T; ++t) {
    const float* yr = y + (long)t * 3 * H;
    const float zz = tanhf(yr[0]), ff = sigmoidf_(yr[H]), oo = sigmoidf_(yr[2 * H]);
    cprev = ff * zz + (1.f - ff) * cprev;
    cp[(long)t * H] = cprev;
    hp[(long)t * ldh] = oo * cprev;
  }
  return cprev;
}

__global__ void __launch_bounds__(128)
qrnn_scan_fwd_kernel(const float* __restrict__ Y, float* __restrict__ h, long ldh,
                     float* __restrict__ Cst, int T, int H) {
  pdl_wait();
  const int n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  qrnn_fwd_seq(Y + (long)n * T * 3 * H + c, h + (long)n * T * ldh + c, ldh,
               Cst + (long)n * T * H + c, T, H, 0.f);
}

// Many streams' scans continued at once (StreamPool): segment blockIdx.y's row {row0, T, slot,
// first} scans rows row0 .. row0+T-1 from state[slot] (0 when first) and writes the state back.
// A slot appears at most once per launch.
__global__ void __launch_bounds__(128)
qrnn_scan_fwd_carry_var_kernel(const float* __restrict__ Y, float* __restrict__ h, long ldh,
                               float* __restrict__ Cst, float* __restrict__ state,
                               const int* __restrict__ tab, int H) {
  pdl_wait();
  const int* row = tab + 4 * blockIdx.y;
  const long row0 = __ldg(row);
  const int T = __ldg(row + 1);
  const long slot = __ldg(row + 2);
  const int first = __ldg(row + 3);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float* st = state + slot * H + c;
  const float c0 = first ? 0.f : *st;
  *st = qrnn_fwd_seq(Y + row0 * 3 * H + c, h + row0 * ldh + c, ldh, Cst + row0 * H + c, T, H,
                     c0);
}

// One sample's sequential backward scan of hidden unit c over its T steps, last to first: y /
// cp / dhp / dy point at its first step, cm0 is the cell state before it and carry the cell-state
// gradient entering from after its last step (both 0 for a whole utterance).  Returns the
// gradient of cm0.  Every step runs the same arithmetic whether it falls in an unrolled group or
// in the remainder, so a backward cut into windows that carry the gradient reproduces the whole
// scan's bits (pase_qrnn_scan_bwd_carry_var).
__device__ __forceinline__ float qrnn_bwd_seq(const float* __restrict__ y,
                                              const float* __restrict__ cp,
                                              const float* __restrict__ dhp, long lddh,
                                              float* __restrict__ dy, int T, int H, float cm0,
                                              float carry) {
  int t = T - 1;
  // the loads do not depend on the recurrence: issue UNROLL time steps of them up front
  for (; t - (UNROLL - 1) >= 0; t -= UNROLL) {
    float z[UNROLL], f[UNROLL], o[UNROLL], c[UNROLL], cm[UNROLL], g[UNROLL];
#pragma unroll
    for (int i = 0; i < UNROLL; ++i) {
      const int tt = t - i;
      const float* yr = y + (long)tt * 3 * H;
      z[i] = yr[0]; f[i] = yr[H]; o[i] = yr[2 * H];
      c[i] = cp[(long)tt * H];
      cm[i] = tt > 0 ? cp[(long)(tt - 1) * H] : cm0;
      g[i] = dhp[(long)tt * lddh];
    }
#pragma unroll
    for (int i = 0; i < UNROLL; ++i) {
      const int tt = t - i;
      const float zz = tanhf(z[i]), ff = sigmoidf_(f[i]), oo = sigmoidf_(o[i]);
      const float dc = g[i] * oo + carry;
      carry = dc * (1.f - ff);
      float* dr = dy + (long)tt * 3 * H;
      dr[0] = dc * ff * (1.f - zz * zz);
      dr[H] = dc * (zz - cm[i]) * ff * (1.f - ff);
      dr[2 * H] = g[i] * c[i] * oo * (1.f - oo);
    }
  }
  for (; t >= 0; --t) {
    const float* yr = y + (long)t * 3 * H;
    const float zz = tanhf(yr[0]), ff = sigmoidf_(yr[H]), oo = sigmoidf_(yr[2 * H]);
    const float ct = cp[(long)t * H];
    const float cm1 = t > 0 ? cp[(long)(t - 1) * H] : cm0;
    const float g = dhp[(long)t * lddh];
    const float dc = g * oo + carry;
    carry = dc * (1.f - ff);
    float* dr = dy + (long)t * 3 * H;
    dr[0] = dc * ff * (1.f - zz * zz);
    dr[H] = dc * (zz - cm1) * ff * (1.f - ff);
    dr[2 * H] = g * ct * oo * (1.f - oo);
  }
  return carry;
}

__global__ void __launch_bounds__(128)
qrnn_scan_bwd_kernel(const float* __restrict__ Y, const float* __restrict__ Cst,
                     const float* __restrict__ dh, long lddh, float* __restrict__ dY, int T,
                     int H) {
  pdl_wait();
  const int n = blockIdx.y;
  const long row0 = (long)n * T;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  qrnn_bwd_seq(Y + row0 * 3 * H + c, Cst + row0 * H + c, dh + row0 * lddh + c, lddh,
               dY + row0 * 3 * H + c, T, H, 0.f, 0.f);
}

// ---- time-segmented scans ----
// The recurrence c_t = f_t z_t + (1-f_t) c_{t-1} is linear in c: a segment of SEG steps maps
// its incoming state to  c_out = A c_in + B  with A = prod(1-f), B = the scan from zero.
// A block owns 32 hidden units x ceil(T/SEG) segments (threadIdx.y = segment): every thread
// scans its segment from zero (gate activations: the expensive part, now 13x more parallel
// at T'=200), the (A, B) pairs meet in shared memory, each thread folds the segments before
// its own (<= 31 FMAs) and corrects its SEG values.  The sequential kernels above keep one
// warp per scheduler busy for 200 dependent steps (45 / 64 us at N=32, H=512); these take
// the chain down to 2 x 16 short steps.
constexpr int SEG = 16;
constexpr int MAX_SEGS = 32;

// One sample's segmented scan: rows row0 .. row0+T-1 of Y / h / Cst; segment threadIdx.y.
__device__ __forceinline__ void qrnn_fwd_seg(const float* __restrict__ Y, float* __restrict__ h,
                                             long ldh, float* __restrict__ Cst, long row0, int T,
                                             int H, float (*sA)[33], float (*sB)[33]) {
  const int lane = threadIdx.x, seg = threadIdx.y;
  const int c = blockIdx.x * 32 + lane;
  const bool live = c < H;
  const int t0 = seg * SEG;
  const int len = (T - t0) < SEG ? (T - t0) : SEG;
  const float* y = Y + (row0 + t0) * 3 * H + c;
  float z[SEG], f[SEG], o[SEG];
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    const bool ok = live && i < len;
    const float* yr = y + (long)i * 3 * H;
    z[i] = ok ? yr[0] : 0.f;
    f[i] = ok ? yr[H] : 0.f;
    o[i] = ok ? yr[2 * H] : 0.f;
  }
  float loc[SEG], pr[SEG];
  float cl = 0.f, P = 1.f;
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    const float zz = tanhf(z[i]), ff = sigmoidf_(f[i]);
    const float keep = (i < len) ? 1.f - ff : 1.f;
    cl = (i < len) ? ff * zz + keep * cl : cl;
    P *= keep;
    loc[i] = cl;
    pr[i] = P;
    o[i] = sigmoidf_(o[i]);
  }
  sA[seg][lane] = P;
  sB[seg][lane] = cl;
  __syncthreads();
  float cin = 0.f;
  for (int s2 = 0; s2 < seg; ++s2) cin = sA[s2][lane] * cin + sB[s2][lane];
  if (!live) return;
  float* hp = h + (row0 + t0) * ldh + c;
  float* cp = Cst + (row0 + t0) * H + c;
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    if (i < len) {
      const float ct = fmaf(pr[i], cin, loc[i]);
      cp[(long)i * H] = ct;
      hp[(long)i * ldh] = o[i] * ct;
    }
  }
}

template <int NSEG_MAX>
__global__ void __launch_bounds__(32 * NSEG_MAX, 1)
qrnn_scan_fwd_seg_kernel(const float* __restrict__ Y, float* __restrict__ h, long ldh,
                         float* __restrict__ Cst, int T, int H) {
  pdl_wait();
  __shared__ float sA[MAX_SEGS][33], sB[MAX_SEGS][33];
  qrnn_fwd_seg(Y, h, ldh, Cst, (long)blockIdx.y * T, T, H, sA, sB);
}

// One sample's segmented backward: rows row0 .. row0+T-1 of Y / Cst / dh, gate gradients to rows
// drow0 .. drow0+T-1 of dY; segment threadIdx.y of blockDim.y.  Segments past the end scan
// nothing and pass the carry through.
__device__ __forceinline__ void qrnn_bwd_seg(const float* __restrict__ Y,
                                             const float* __restrict__ Cst,
                                             const float* __restrict__ dh, long lddh,
                                             float* __restrict__ dY, long row0, long drow0, int T,
                                             int H, float (*sA)[33], float (*sB)[33]) {
  const int lane = threadIdx.x, seg = threadIdx.y, nseg = blockDim.y;
  const int c = blockIdx.x * 32 + lane;
  const bool live = c < H;
  const int t0 = seg * SEG;
  const int len = (T - t0) < SEG ? (T - t0) : SEG;
  const float* y = Y + (row0 + t0) * 3 * H + c;
  const float* cp = Cst + (row0 + t0) * H + c;
  const float* dhp = dh + (row0 + t0) * lddh + c;
  float* dy = dY + (drow0 + t0) * 3 * H + c;
  float z[SEG], f[SEG], o[SEG], cs[SEG], g[SEG];
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    const bool ok = live && i < len;
    const float* yr = y + (long)i * 3 * H;
    z[i] = ok ? yr[0] : 0.f;
    f[i] = ok ? yr[H] : 0.f;
    o[i] = ok ? yr[2 * H] : 0.f;
    cs[i] = ok ? cp[(long)i * H] : 0.f;
    g[i] = ok ? dhp[(long)i * lddh] : 0.f;
  }
  const float cm0 = (live && t0 > 0 && len > 0) ? cp[-(long)H] : 0.f;       // c_{t0-1}
  // right-to-left local scan with zero incoming carry; z[] / f[] are overwritten by the
  // coefficients of the correction pass (dz = dc kz, df = dc kf), cs[] / o[] by (local dc, Q)
  float carry = 0.f, Q = 1.f;
#pragma unroll
  for (int i = SEG - 1; i >= 0; --i) {
    const float zz = tanhf(z[i]), ff = sigmoidf_(f[i]), oo = sigmoidf_(o[i]);
    const float cm = i > 0 ? cs[i - 1] : cm0;
    const float ct = cs[i];
    const bool in = i < len;
    const float dc = in ? fmaf(g[i], oo, carry) : 0.f;
    if (live && in) dy[(long)i * 3 * H + 2 * H] = g[i] * ct * oo * (1.f - oo);
    z[i] = ff * (1.f - zz * zz);                 // kz
    f[i] = (zz - cm) * ff * (1.f - ff);          // kf
    cs[i] = dc;                                  // local dc
    o[i] = Q;                                    // prod_{s>t}(1-f_s) inside the segment
    if (in) {
      carry = dc * (1.f - ff);
      Q *= (1.f - ff);
    }
  }
  sA[seg][lane] = Q;
  sB[seg][lane] = carry;
  __syncthreads();
  float kin = 0.f;                               // carry entering from the right
  for (int s2 = nseg - 1; s2 > seg; --s2) kin = sA[s2][lane] * kin + sB[s2][lane];
  if (!live) return;
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    if (i < len) {
      const float dc = fmaf(o[i], kin, cs[i]);
      dy[(long)i * 3 * H] = dc * z[i];
      dy[(long)i * 3 * H + H] = dc * f[i];
    }
  }
}

template <int NSEG_MAX>
__global__ void __launch_bounds__(32 * NSEG_MAX, 1)
qrnn_scan_bwd_seg_kernel(const float* __restrict__ Y, const float* __restrict__ Cst,
                         const float* __restrict__ dh, long lddh, float* __restrict__ dY, int T,
                         int H) {
  pdl_wait();
  __shared__ float sA[MAX_SEGS][33], sB[MAX_SEGS][33];
  const int n = blockIdx.y;
  const long row0 = (long)n * T;
  qrnn_bwd_seg(Y, Cst, dh, lddh, dY, row0, row0, T, H, sA, sB);
}

// Segments per block of the time-segmented kernels for T time steps (the template width: 16,
// 24 or 32), or 0 above MAX_SEGS segments, where only the sequential kernels apply.
inline int seg_width(int T) {
  const int nseg = (T + SEG - 1) / SEG;
  return nseg <= 16 ? 16 : nseg <= 24 ? 24 : nseg <= MAX_SEGS ? MAX_SEGS : 0;
}

// Packed variable-length forms: blockIdx.y = utterance, tab row {row0, T}.  Each utterance
// runs the algorithm its own length selects (seg_width), so it gets the bits of a B=1 scan:
// the segmented kernel skips utterances longer than MAX_SEGS segments, the sequential one the
// others.  Segments past an utterance's end scan nothing and pass the state through.
__global__ void __launch_bounds__(32 * MAX_SEGS, 1)
qrnn_scan_fwd_seg_var_kernel(const float* __restrict__ Y, float* __restrict__ h, long ldh,
                             float* __restrict__ Cst, const int* __restrict__ tab, int H) {
  pdl_wait();
  __shared__ float sA[MAX_SEGS][33], sB[MAX_SEGS][33];
  const int T = __ldg(tab + 2 * blockIdx.y + 1);
  if (T > SEG * MAX_SEGS) return;
  qrnn_fwd_seg(Y, h, ldh, Cst, __ldg(tab + 2 * blockIdx.y), T, H, sA, sB);
}

__global__ void __launch_bounds__(128)
qrnn_scan_fwd_seq_var_kernel(const float* __restrict__ Y, float* __restrict__ h, long ldh,
                             float* __restrict__ Cst, const int* __restrict__ tab, int H) {
  pdl_wait();
  const int T = __ldg(tab + 2 * blockIdx.y + 1);
  const long row0 = __ldg(tab + 2 * blockIdx.y);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (T <= SEG * MAX_SEGS || c >= H) return;
  qrnn_fwd_seq(Y + row0 * 3 * H + c, h + row0 * ldh + c, ldh, Cst + row0 * H + c, T, H, 0.f);
}

// Packed variable-length backward: blockIdx.y = utterance, tab row {row0, T, drow0}: rows row0 ..
// row0+T-1 of Y / Cst / dh are one utterance, its gate gradients go to rows drow0 .. drow0+T-1
// of dY and row drow0+T of dY is written zero (the QRNN input's rows, one separator row per
// utterance: DESIGN.md section 18).  As in the forward, each utterance runs the body its own T
// selects (qrnn_bwd_seg or qrnn_bwd_seq).
__global__ void __launch_bounds__(32 * MAX_SEGS, 1)
qrnn_scan_bwd_seg_var_kernel(const float* __restrict__ Y, const float* __restrict__ Cst,
                             const float* __restrict__ dh, long lddh, float* __restrict__ dY,
                             const int* __restrict__ tab, int H) {
  pdl_wait();
  __shared__ float sA[MAX_SEGS][33], sB[MAX_SEGS][33];
  const int* r = tab + 3 * blockIdx.y;
  const int T = __ldg(r + 1);
  if (T > SEG * MAX_SEGS) return;
  const long row0 = __ldg(r), drow0 = __ldg(r + 2);
  const int c = blockIdx.x * 32 + threadIdx.x;
  if (c < H && threadIdx.y == 0) {
    float* zr = dY + (drow0 + T) * 3 * H + c;
    zr[0] = 0.f; zr[H] = 0.f; zr[2 * H] = 0.f;
  }
  qrnn_bwd_seg(Y, Cst, dh, lddh, dY, row0, drow0, T, H, sA, sB);
}

__global__ void __launch_bounds__(128)
qrnn_scan_bwd_seq_var_kernel(const float* __restrict__ Y, const float* __restrict__ Cst,
                             const float* __restrict__ dh, long lddh, float* __restrict__ dY,
                             const int* __restrict__ tab, int H) {
  pdl_wait();
  const int* r = tab + 3 * blockIdx.y;
  const int T = __ldg(r + 1);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (T <= SEG * MAX_SEGS || c >= H) return;
  const long row0 = __ldg(r), drow0 = __ldg(r + 2);
  float* dy = dY + drow0 * 3 * H + c;
  qrnn_bwd_seq(Y + row0 * 3 * H + c, Cst + row0 * H + c, dh + row0 * lddh + c, lddh, dy, T, H,
               0.f, 0.f);
  dy[(long)T * 3 * H] = 0.f; dy[(long)T * 3 * H + H] = 0.f; dy[(long)T * 3 * H + 2 * H] = 0.f;
}

// Backward of one window's carried scan (WaveFe.encode_long): tab row {row0, T, drow0, c0, cn,
// slot} per window (blockIdx.y).  Rows row0 .. row0+T-1 of Y / Cst / dh are the window's frames,
// of which c0 .. c0+cn-1 (its crop) were scanned from state[slot]; the gate gradients of the crop
// go to rows drow0+c0 .. of dY, every other row of drow0 .. drow0+T (the separator included) is
// written zero.  The scan starts from the cell-state gradient dstate[slot] (the next window's
// gradient of this window's last state) and leaves there the gradient of state[slot].
__global__ void __launch_bounds__(128)
qrnn_scan_bwd_carry_var_kernel(const float* __restrict__ Y, const float* __restrict__ Cst,
                               const float* __restrict__ dh, long lddh, float* __restrict__ dY,
                               const float* __restrict__ state, float* __restrict__ dstate,
                               const int* __restrict__ tab, int H) {
  pdl_wait();
  const int* r = tab + 6 * blockIdx.y;
  const long row0 = __ldg(r), drow0 = __ldg(r + 2), slot = __ldg(r + 5);
  const int T = __ldg(r + 1), c0 = __ldg(r + 3), cn = __ldg(r + 4);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float* dy = dY + drow0 * 3 * H + c;
  for (int t = 0; t <= T; ++t) {
    if (t >= c0 && t < c0 + cn) continue;
    float* dr = dy + (long)t * 3 * H;
    dr[0] = 0.f; dr[H] = 0.f; dr[2 * H] = 0.f;
  }
  float* ds = dstate + slot * H + c;
  *ds = qrnn_bwd_seq(Y + (row0 + c0) * 3 * H + c, Cst + (row0 + c0) * H + c,
                     dh + (row0 + c0) * lddh + c, lddh, dy + (long)c0 * 3 * H, cn, H,
                     state[slot * H + c], *ds);
}

// Launches a uniform (N, T) scan: seg16 / seg24 / seg32, the time-segmented kernel of the width
// seg_width(T) selects, with one (32, ceil(T/SEG)) block per 32 hidden units and sample, or seq,
// the sequential kernel, with one thread per hidden unit and sample when T is longer.
template <typename... KArgs, typename... Args>
int launch_scan(const char* name, void (*seg16)(KArgs...), void (*seg24)(KArgs...),
                void (*seg32)(KArgs...), void (*seq)(KArgs...), int N, int T, int H,
                cudaStream_t st, Args... args) {
  const int width = seg_width(T);
  if (width)
    PASE_LAUNCH(width == 16 ? seg16 : width == 24 ? seg24 : seg32, dim3((H + 31) / 32, N),
                dim3(32, (T + SEG - 1) / SEG), 0, st, args...);
  else
    PASE_LAUNCH(seq, dim3((H + 127) / 128, N), 128, 0, st, args...);
  PASE_LAUNCH_CHECK(name);
  return PASE_OK;
}

}  // namespace

extern "C" {

int pase_qrnn_scan_fwd_var(const float* Y, float* h, long ldh, float* Cst, const int* tab,
                           int nseg, int H, void* stream) {
  PASE_CHECK_ARG(Y && h && Cst && tab, "pase_qrnn_scan_fwd_var: null pointer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && H > 0 && ldh >= H,
                 "pase_qrnn_scan_fwd_var: nseg=%d H=%d ldh=%ld", nseg, H, ldh);
  cudaStream_t st = (cudaStream_t)stream;
  PASE_LAUNCH((qrnn_scan_fwd_seg_var_kernel), dim3((H + 31) / 32, nseg), dim3(32, MAX_SEGS), 0,
              st, Y, h, ldh, Cst, tab, H);
  PASE_LAUNCH_CHECK("pase_qrnn_scan_fwd_var");
  PASE_LAUNCH((qrnn_scan_fwd_seq_var_kernel), dim3((H + 127) / 128, nseg), 128, 0, st, Y, h, ldh,
              Cst, tab, H);
  PASE_LAUNCH_CHECK("pase_qrnn_scan_fwd_var");
  return PASE_OK;
}

int pase_qrnn_scan_fwd(const float* Y, float* h, long ldh, float* Cst, int N, int T, int H,
                       void* stream) {
  PASE_CHECK_ARG(Y && h && Cst, "pase_qrnn_scan_fwd: null pointer");
  PASE_CHECK_ARG(N > 0 && T > 0 && H > 0, "pase_qrnn_scan_fwd: N=%d T=%d H=%d", N, T, H);
  PASE_CHECK_ARG(ldh >= H, "pase_qrnn_scan_fwd: ldh=%ld < H=%d", ldh, H);
  return launch_scan("pase_qrnn_scan_fwd", qrnn_scan_fwd_seg_kernel<16>,
                     qrnn_scan_fwd_seg_kernel<24>, qrnn_scan_fwd_seg_kernel<MAX_SEGS>,
                     qrnn_scan_fwd_kernel, N, T, H, (cudaStream_t)stream, Y, h, ldh, Cst, T, H);
}

int pase_qrnn_scan_fwd_carry_var(const float* Y, float* h, long ldh, float* Cst, float* state,
                                 const int* tab, int nseg, int H, void* stream) {
  PASE_CHECK_ARG(Y && h && Cst && state && tab, "pase_qrnn_scan_fwd_carry_var: null pointer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && H > 0 && ldh >= H,
                 "pase_qrnn_scan_fwd_carry_var: nseg=%d H=%d ldh=%ld", nseg, H, ldh);
  PASE_LAUNCH((qrnn_scan_fwd_carry_var_kernel), dim3((H + 127) / 128, nseg), 128, 0,
              (cudaStream_t)stream, Y, h, ldh, Cst, state, tab, H);
  PASE_LAUNCH_CHECK("pase_qrnn_scan_fwd_carry_var");
  return PASE_OK;
}

int pase_qrnn_scan_bwd(const float* Y, const float* Cst, const float* dh, long lddh, float* dY,
                       int N, int T, int H, void* stream) {
  PASE_CHECK_ARG(Y && Cst && dh && dY, "pase_qrnn_scan_bwd: null pointer");
  PASE_CHECK_ARG(N > 0 && T > 0 && H > 0, "pase_qrnn_scan_bwd: N=%d T=%d H=%d", N, T, H);
  PASE_CHECK_ARG(lddh >= H, "pase_qrnn_scan_bwd: lddh=%ld < H=%d", lddh, H);
  return launch_scan("pase_qrnn_scan_bwd", qrnn_scan_bwd_seg_kernel<16>,
                     qrnn_scan_bwd_seg_kernel<24>, qrnn_scan_bwd_seg_kernel<MAX_SEGS>,
                     qrnn_scan_bwd_kernel, N, T, H, (cudaStream_t)stream, Y, Cst, dh, lddh, dY, T,
                     H);
}

int pase_qrnn_scan_bwd_var(const float* Y, const float* Cst, const float* dh, long lddh, float* dY,
                           const int* tab, int nseg, int H, void* stream) {
  PASE_CHECK_ARG(Y && Cst && dh && dY && tab, "pase_qrnn_scan_bwd_var: null pointer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && H > 0 && lddh >= H,
                 "pase_qrnn_scan_bwd_var: nseg=%d H=%d lddh=%ld", nseg, H, lddh);
  cudaStream_t st = (cudaStream_t)stream;
  PASE_LAUNCH((qrnn_scan_bwd_seg_var_kernel), dim3((H + 31) / 32, nseg), dim3(32, MAX_SEGS), 0,
              st, Y, Cst, dh, lddh, dY, tab, H);
  PASE_LAUNCH_CHECK("pase_qrnn_scan_bwd_var");
  PASE_LAUNCH((qrnn_scan_bwd_seq_var_kernel), dim3((H + 127) / 128, nseg), 128, 0, st, Y, Cst, dh,
              lddh, dY, tab, H);
  PASE_LAUNCH_CHECK("pase_qrnn_scan_bwd_var");
  return PASE_OK;
}

int pase_qrnn_scan_bwd_carry_var(const float* Y, const float* Cst, const float* dh, long lddh,
                                 float* dY, const float* state, float* dstate, const int* tab,
                                 int nseg, int H, void* stream) {
  PASE_CHECK_ARG(Y && Cst && dh && dY && state && dstate && tab,
                 "pase_qrnn_scan_bwd_carry_var: null pointer");
  PASE_CHECK_ARG(nseg > 0 && nseg <= 65535 && H > 0 && lddh >= H,
                 "pase_qrnn_scan_bwd_carry_var: nseg=%d H=%d lddh=%ld", nseg, H, lddh);
  PASE_LAUNCH((qrnn_scan_bwd_carry_var_kernel), dim3((H + 127) / 128, nseg), 128, 0,
              (cudaStream_t)stream, Y, Cst, dh, lddh, dY, state, dstate, tab, H);
  PASE_LAUNCH_CHECK("pase_qrnn_scan_bwd_carry_var");
  return PASE_OK;
}

int pase_qrnn_scan_plan(int T, int* out1) {
  PASE_CHECK_ARG(out1 && T > 0, "pase_qrnn_scan_plan: bad args");
  out1[0] = seg_width(T);
  return PASE_OK;
}

}  // extern "C"
