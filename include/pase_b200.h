/*
 * pase_b200 -- C-ABI of the native PASE/PASE+ hot path (H100, sm_90a).
 *
 * The reference (santi-pdp/pase) is pure Python/PyTorch and has no FFI; the
 * boundary a maintainer binds is therefore this library, loaded with ctypes
 * from the Python shim (pase_b200/_lib.py) that mirrors
 * pase.models.frontend.wf_builder / pase.models.pase.pase.  Every entry point
 * below replaces one library call (cuDNN / cuBLAS / ATen / torchqrnn) that the
 * reference issues on this path; the reference call site is cited per entry
 * as /root/reference/<file>:<line>.
 *
 * Conventions
 *   - the packed and windowed entry points (*_var, pase_stream_gather) give each table row
 *     (utterance, segment or stream) one grid row: nseg / nrow must be in 1..65535, anything
 *     else is refused (PASE_ERR_ARG) before a launch;
 *   - all pointers are DEVICE pointers into buffers owned by the caller
 *     (PyTorch caching allocator); the library allocates nothing persistent;
 *   - activations are channel-last: (sample, time, channel), fp32;
 *   - `stream` is a cudaStream_t passed as void*;
 *   - return value 0 = ok, otherwise a negative pase error code or a positive
 *     cudaError_t; pase_last_error() returns a thread-local message.
 */
#ifndef PASE_B200_H
#define PASE_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define PASE_OK 0
#define PASE_ERR_ARG (-1)
#define PASE_ERR_UNSUPPORTED (-2)

const char* pase_last_error(void);
int pase_version(void);
/* Device properties the host side sizes grids with: out[0]=SM count,
 * out[1]=cc major, out[2]=cc minor, out[3]=max opt-in smem per block. */
int pase_device_info(int* out4);

/* ---- GEMM family (replaces F.conv1d / nn.Conv1d / nn.Linear /
 * nn.ConvTranspose1d and their backward: modules.py:932,1072,
 * frontend.py:195,244-262, minions.py:494-524, torchqrnn linear) -----------
 *
 * pase_gemm_nt:  C[map(m), n] (+)= alpha * sum_k A[m*lda + k] * B[n*ldb + k] + bias[n]
 *   A may be an OVERLAPPING-row view (lda < K): row m of a strided 1-D
 *   convolution's implicit im2col matrix is K contiguous floats of the padded
 *   channel-last activation starting at m*lda.
 *   Row map: g = m / rows_in, u = m % rows_in.  Element (u, n) is valid iff
 *   u*fold + n/(N/fold) < t_valid; it is stored at row g*rows_out + u.
 *   colsum/colsumsq (double[N], may be NULL) accumulate the per-column sum and
 *   sum of squares of the valid outputs (BatchNorm batch statistics).
 *   This entry point computes in fp32 FFMA; pase_tc_gemm_nt is the tensor-core variant.
 */
int pase_gemm_nt(const float* A, long lda, const float* B, long ldb,
                 float* C, long ldc, int M, int N, int K,
                 float alpha, const float* bias,
                 int rows_in, int t_valid, int rows_out, int fold,
                 double* colsum, double* colsumsq, int accumulate,
                 void* stream);

/* pase_gemm_tn:  C[i, j] (+)= alpha * sum_r A[rowA(r)*lda + i] * B[rowB(r)*ldb + j]
 *   r in [0, groups*rows_per_group): g = r / rows_per_group, u = r % rows_per_group,
 *   rowA = g*pitchA + offA + u, rowB = g*pitchB + offB + u.
 *   (weight gradients: reduction over samples x time.) */
int pase_gemm_tn(const float* A, long lda, int pitchA, int offA,
                 const float* B, long ldb, int pitchB, int offB,
                 float* C, long ldc, int I, int J,
                 int groups, int rows_per_group,
                 float alpha, int accumulate, void* stream);


/* ---- tensor-core (wgmma / TMA) GEMMs ---------------------------------------
 * Same contract as pase_gemm_nt / pase_gemm_tn, computed with wgmma
 * instructions and fp32 accumulation in registers.  `mode` selects the
 * operand element type and the numerics:
 *   0  TF32   : fp32 operands read as tf32, one pass;
 *   1  3xTF32 : fp32 operands pre-split by pase_split_tf32 into exactly
 *               representable hi/lo parts = fp32-equivalent products;
 *   2  BF16   : bf16 operands, one pass at twice the TF32 rate;
 *   3  3xF16  : fp16 operand pairs x = hi + 2^-11 lo' (pase_split_f16 or the
 *               producing kernel) = fp32-equivalent products at half the tensor
 *               time and operand bytes of 3xTF32; operands must fit fp16's
 *               range (gradients are pre-scaled by a power of two).
 * Ahi/Alo/Bhi/Blo point to fp32 (modes 0,1), bf16 (2) or fp16 (3) arrays; the
 * lo pointers are NULL outside modes 1 and 3.
 * A is a plain 2-D tensor [a_rows x R] (R elements per folded row, R*elemsize
 * a multiple of 128 bytes): element (m, k) is read at row m + k/R, column k%R.
 * alpha_dev (may be NULL): device scalar multiplied into alpha (undoes the
 * power-of-two scale of a pre-scaled gradient operand without a host sync).
 * c_bf16 != 0: C is a bf16 array (no accumulate); otherwise fp32. */
int pase_split_tf32(const float* x, float* hi, float* lo, long n, void* stream);
int pase_tc_gemm_nt(const void* Ahi, const void* Alo, long a_rows, int R,
                    const void* Bhi, const void* Blo, long ldb,
                    void* C, long ldc, int M, int N, int K, float alpha,
                    const float* alpha_dev, const float* bias,
                    int rows_in, int t_valid, int rows_out, int fold,
                    double* colsum, double* colsumsq, int accumulate, int mode, int c_bf16,
                    void* stream);
/* Packed variable-length forms of pase_gemm_nt (FFMA) and pase_tc_gemm_nt (inference: alpha 1,
 * no statistics, no accumulation).  Utterance i's GEMM rows are contiguous; each one's padded
 * operand starts on a folded-row boundary, so a row reads the K elements of its own utterance
 * and the loads are those of the uniform kernels.  Only the epilogue's row map differs: var_tab
 * (DEVICE, 3*nvar+1 ints) = row0[0..nvar] (first GEMM row of each utterance, ascending; row0[nvar]
 * = rows in use, <= M), orow0[nvar] (first output row), t_valid[nvar].  Row m of utterance i
 * (u = m - row0[i]) stores element (u, n) at output row orow0[i] + u iff
 * u*fold + n/(N/fold) < t_valid[i]; rows >= row0[nvar] store nothing. */
int pase_gemm_nt_var(const float* A, long lda, const float* B, long ldb, float* C, long ldc,
                     int M, int N, int K, const float* bias, const int* var_tab, int nvar,
                     int fold, void* stream);
int pase_tc_gemm_nt_var(const void* Ahi, const void* Alo, long a_rows, int R,
                        const void* Bhi, const void* Blo, long ldb, void* C, long ldc,
                        int M, int N, int K, const float* bias, const int* var_tab, int nvar,
                        int fold, int mode, int c_bf16, void* stream);
/* The two packed GEMMs above with train-mode BatchNorm column statistics (WaveFe.
 * encode_packed_train, DESIGN.md section 19; FeBlock's conv -> BatchNorm1d,
 * pase/models/modules.py:1014-1077): colsum[n] += sum C(m, n), colsumsq[n] += sum C(m, n)^2
 * (DEVICE, double[N], N <= 4096) over exactly the elements the row map stores, so over the
 * valid frames of every utterance and nothing else; in the folded sinc layer column n is
 * virtual channel n of the fold, summed by pase_bn_finalize.  The sums are those of the uniform
 * kernels' epilogues (fp32 per tile, fp64 across tiles); both launches of a partial last round
 * take part. */
int pase_gemm_nt_var_stats(const float* A, long lda, const float* B, long ldb, float* C,
                           long ldc, int M, int N, int K, const float* bias, const int* var_tab,
                           int nvar, int fold, double* colsum, double* colsumsq, void* stream);
int pase_tc_gemm_nt_var_stats(const void* Ahi, const void* Alo, long a_rows, int R,
                              const void* Bhi, const void* Blo, long ldb, void* C, long ldc,
                              int M, int N, int K, const float* bias, const int* var_tab,
                              int nvar, int fold, double* colsum, double* colsumsq, int mode,
                              int c_bf16, void* stream);
/* How pase_tc_gemm_nt / pase_tc_gemm_nt_var cover an M x N output on `sms` SMs (host only):
 * out4 = {bn, bulk_m, tail_bn, tail_pieces}.  One launch of 128 x bn tiles takes rows
 * [0, bulk_m); when the tiles leave a partial last round, a second launch takes rows
 * [bulk_m, M) at every column in tail_pieces tiles of 128 x tail_bn (tail_bn 0: no second
 * launch, bulk_m = M).  K is never split, so the results do not depend on the plan. */
int pase_tc_gemm_nt_plan(int M, int N, int sms, int* out4);
int pase_tc_gemm_tn(const void* Ahi, const void* Alo, long lda, int pitchA, int offA,
                    const void* Bhi, const void* Blo, int R, int pitchB, long b_rows_total,
                    float* C, long ldc, int I, int J, int groups, int rows_per_group,
                    float alpha, const float* alpha_dev, int accumulate, int mode, void* stream);
/* How pase_tc_gemm_tn splits the reduction of this shape on the current device (host only):
 * out2 = {splits, chunks_per_split}; a chunk is 32 reduction rows in modes 0/1, 64 in 2/3. */
int pase_tc_gemm_tn_plan(int I, int J, int groups, int rows_per_group, int mode, int* out2);

/* ---- operand-format conversions for GEMM modes 2 / 3 (small tensors) -------- */
/* dst (bf16) = rn(x) */
int pase_cast_bf16(const float* x, void* dst, long n, void* stream);
/* amax[0] = max(amax[0], max|x|)  (caller zeroes amax once per use) */
int pase_absmax(const float* x, long n, float* amax, void* stream);
/* fp16 pair of s*x: hi = rn_f16(s x), lo = rn_f16((s x - hi) 2^11); s = 1 when amax is
 * NULL, else the power of two placing amax[0] below 2^14; scale_out = {1/s, s} */
int pase_split_f16(const float* x, void* hi, void* lo, long n, const float* amax,
                   float* scale_out, void* stream);

/* amax[0] = max(amax[0], max_r ||X[r, :cols]||_2)   (Cauchy-Schwarz bound of a GEMM output) */
int pase_rownorm_max(const float* X, long ld, long rows, int cols, float* amax, void* stream);
/* scale_out = {1/s, s}: the power of two placing a[0]*a[1] + a[2] + a[3] below 2^14 */
int pase_bound_scale(const float* a4, float* scale_out, void* stream);

/* ---- fused regression head (MLPMinion output layer + ContextualizedLoss MSE:
 * minions.py:494-524, losses.py:15-37, GEMM mode 3) ------------------------
 * residual[m, n] = sum_k A[m,k] B[n,k] + bias[n] - label[b][n/r][t + n%r - r/2]
 * (m = b*T + t; zero outside [0,T)): never stored as fp32 -- Rhi/Rlo receive the fp16
 * pair of s * residual ([M x ldr], ldr % 128 == 0, columns >= N zero), the operand of
 * the two backward GEMMs; loss_acc += sum residual^2; db_acc[n] += sum_m residual[m,n].
 * scale = device {1/s, s} (pase_bound_scale of the Cauchy-Schwarz bound).
 * Loss only (no gradient will be taken): Rhi, Rlo and db_acc all NULL -- only loss_acc is
 * written, with the same sum; scale may then be NULL too. */
int pase_tc_gemm_nt_ctxmse(const void* Ahi, const void* Alo, long a_rows, int R,
                           const void* Bhi, const void* Blo, long ldb,
                           void* Rhi, void* Rlo, long ldr, int M, int N, int K,
                           const float* bias, const float* label, int B, int F, int T, int r,
                           const float* scale, double* loss_acc, double* db_acc, void* stream);

/* ---- weight re-layout (implicit-GEMM operand preparation) ---------------- */
/* (Cout,Cin,k) -> Wt[co, j*Cin+ci]                      (forward operand)   */
int pase_conv_w_to_fwd(const float* W, float* Wt, int Cout, int Cin, int k, void* stream);
/* (Cout,Cin,k) -> Wd[p*Cin+ci, v*Cout+co] = W[co,ci,s*(taps-1-v)+p] or 0    */
int pase_conv_w_to_dgrad(const float* W, float* Wd, int Cout, int Cin, int k,
                         int s, int taps, void* stream);
/* dWt[co, j*Cin+ci] -> dW (Cout,Cin,k)                                      */
int pase_conv_w_from_fwd(const float* dWt, float* dW, int Cout, int Cin, int k, void* stream);
/* The three re-layouts above for EVERY conv block of a step in one launch (the per-layer
 * calls are ~4 us each and there are 35 of them per PASE+ step).  table: device array of
 * njobs x 12 int64 {src, dst, hi, lo, Cout, Cin, k, s, taps, start, count, 0}; start = prefix
 * sum of count (flat element index space of size total); op 0 = to_fwd, 1 = to_dgrad,
 * 2 = from_fwd (dst is then an element offset into dst_base).  hi/lo != 0 additionally write
 * the 3xTF32 weight split (as pase_split_tf32 with an explicit hi).  op 3..5 = the same
 * three through shared-memory tiles (coalesced reads and writes): `total` is then the number
 * of thread blocks, table[.., 11] the job's first block; blocks per job = Cout (ops 3, 5) or
 * (Cout/32)*(Cin/8) (op 4); needs Cout % 32 == 0, Cin % 8 == 0 and (Cin+1)*k <= 12000.
 * fmt selects what hi/lo receive: 0 = the 3xTF32 split (fp32), 1 = bf16 copy in hi,
 * 2 = fp16 pair (hi, lo' = (v-hi)*2^11); dst (fp32) may be 0 when only hi/lo are wanted. */
int pase_conv_w_batch(const long* table, int njobs, long total, int op, float* dst_base,
                      int fmt, void* stream);
/* njobs strided 2-D copies in one launch: table rows of 6 int64 {src, dst, rows, cols,
 * src_ld, dst_ld} (device pointers, fp32 elements); total = sum rows*cols.  Used to place
 * every small gradient of a step into the flat gradient buffer (pase_b200/optim.py). */
int pase_scatter_copy(const long* table, int njobs, long total, void* stream);
/* ConvTranspose1d weight (Cin,Cout,k) -> Wu[p*Cout+co, v*Cin+ci] =
 * W[ci,co,s*(taps-1-v)+p] or 0 (forward operand of the transposed conv)     */
int pase_deconv_w_to_fwd(const float* W, float* Wu, int Cin, int Cout, int k,
                         int s, int taps, void* stream);
/* dWu -> dW (Cin,Cout,k) (inverse gather of the above)                      */
int pase_deconv_w_from_fwd(const float* dWu, float* dW, int Cin, int Cout, int k,
                           int s, int taps, void* stream);
/* dst (cols x ldd) = src(rows x cols)^T, zero-padding columns rows..ldd-1 */
int pase_transpose_pad(const float* src, long lds, float* dst, long ldd, int rows, int cols,
                       void* stream);
/* ConvTranspose1d weight -> backward-data operand Wb[ci, j*Cout+co]=W[ci,co,j] */
int pase_deconv_w_to_bwd(const float* W, float* Wb, int Cin, int Cout, int k, void* stream);

/* ---- SincConv_fast band-pass generator (modules.py:868-918) -------------- */
/* low_hz_,band_hz_ (C) + host-precomputed n_ and window_ (k/2 each) ->
 * polyphase forward operand Wp[(p*C+co), kk] = filt[co][kk-p] (0 outside),
 * p < fold, kk < Kv; also writes filt (C,k) if non-NULL. */
int pase_sinc_make(const float* low_hz, const float* band_hz,
                   const float* n_, const float* window_,
                   float* filt, float* Wp, int C, int k, int fold, int Kv,
                   float min_low, float min_band, float sr, void* stream);
/* dWp -> d low_hz_, d band_hz_ (through abs / clamp / sin) */
int pase_sinc_grad(const float* dWp, const float* low_hz, const float* band_hz,
                   const float* n_, const float* window_,
                   float* dlow, float* dband, int C, int k, int fold, int Kv,
                   float min_low, float min_band, float sr, void* stream);

/* ---- padding / BatchNorm / PReLU (F.pad reflect, nn.BatchNorm1d, nn.PReLU:
 * modules.py:924-928,1071-1075,79,111-113) --------------------------------- */
/* Storage formats of activation-sized tensors (`*_fmt` arguments; `*_bf16` flags
 * are 0 = fp32, 1 = bf16):
 *   0 fp32 (optionally with a tf32-residual twin `*_lo` for GEMM mode 1),
 *   1 bf16 (GEMM mode 2),
 *   2 fp16 pair: dst = hi = rn_f16(x), dst_lo = lo' = rn_f16((x-hi)*2^11) (GEMM mode 3). */
/* (N,T) waveform -> reflect-padded rows of pitch `pitch` elements */
int pase_reflect_pad_wave(const float* x, void* dst, void* dst_lo, int dst_fmt, int N, int T,
                          int padL, int padR, long pitch, void* stream);
/* Packed variable-length form: tab (DEVICE, nseg rows of 3 ints) {x_off, T, dst_off}: utterance
 * x[x_off, +T) reflect-padded into dst[dst_off, +T+padL+padR); max_T >= every T; nseg <= 65535. */
int pase_reflect_pad_wave_var(const float* x, const int* tab, int nseg, int max_T, void* dst,
                              void* dst_lo, int dst_fmt, int padL, int padR, void* stream);

/* ---- input (waveform) gradient of the sinc layer: the input gradients of F.conv1d and
 * F.pad(mode='reflect') in SincConv_fast.forward (modules.py:922-928).  The transposed
 * band-pass convolution is one polyphase NT GEMM (pase_gemm_nt / pase_tc_gemm_nt):
 *   dxpad[n, fold v + p] = sum_{r<rows, q<fold, co<C} dyh[n, fold (v + r) + q, co] Wdg[p, (r,q,co)]
 * with H = (rows-1) fold the left halo (DESIGN.md section 17). ---------------------------- */
/* dy (N samples of src_frames frames x C channels, esz-byte elements, any operand format; lo
 * twins optional, both or neither) -> dyh: N samples of dst_frames frames, frame e = dy frame
 * e - halo, zero outside [0, T_out) -- so no sample reads its neighbours' frames. */
int pase_sinc_dgrad_pack(const void* src, const void* src_lo, void* dst, void* dst_lo, int esz,
                         int N, int C, int T_out, long src_frames, int halo, long dst_frames,
                         void* stream);
/* band-pass bank filt (C,k) (pase_sinc_make) -> banded operand Wdg (fold x rows*fold*C):
 * Wdg[p, (r*fold+q)*C+co] = filt[co][H+p-fold*r-q] inside [0,k), else 0; H = (rows-1)*fold. */
int pase_sinc_dgrad_weight(const float* filt, float* Wdg, int C, int k, int fold, int rows,
                           void* stream);
/* adjoint of pase_reflect_pad_wave: dx[n,t] = dpad[n,t+padL] + [1<=t<=padL] dpad[n,padL-t]
 * + [T-1-padR<=t<=T-2] dpad[n,padL+2(T-1)-t]  (dpad rows of pitch `pitch`, dx (N,T) fp32) */
int pase_reflect_fold_wave(const float* dpad, long pitch, float* dx, int N, int T, int padL,
                           int padR, void* stream);
/* Packed form of pase_reflect_fold_wave: tab (DEVICE, nseg rows of 3 ints) {x_off, T, dst_off}
 * (pase_reflect_pad_wave_var's table): dx[x_off + t] from dpad[dst_off ..]; max_T >= every T. */
int pase_reflect_fold_wave_var(const float* dpad, const int* tab, int nseg, int max_T, float* dx,
                               int padL, int padR, void* stream);
/* One window of a recording's backward (WaveFe.encode_long): dx[x0 + t] += the fold of the
 * window's padded gradient dpad (T + padL + padR floats) at t, for t < T.  The mirrored pad
 * gradient is added on the left only when fold_l != 0 and on the right only when fold_r != 0 (the
 * sides where the window's reflect pad is the recording's own); x0 is a 64-bit offset.  Windows
 * overlap, so dx accumulates: run them one after the other, never concurrently. */
int pase_reflect_fold_wave_acc(const float* dpad, float* dx, long x0, int T, int padL, int padR,
                               int fold_l, int fold_r, void* stream);
/* batch statistics -> per-channel affine; updates running stats (training) */
int pase_bn_finalize(const double* colsum, const double* colsumsq, int C, int fold,
                     double count, const float* gamma, const float* beta,
                     float* running_mean, float* running_var, float momentum, float eps,
                     float* mean, float* invstd, float* scale, float* shift, void* stream);
int pase_bn_eval_affine(const float* running_mean, const float* running_var,
                        const float* gamma, const float* beta, int C, float eps,
                        float* mean, float* invstd, float* scale, float* shift, void* stream);
/* a = PReLU(y*scale+shift) written with reflect halo into the next layer's
 * padded operand buffer (format dst_fmt), plus mean-pooled dense-skip
 * accumulation into the fp32 `pool` matrix (frontend.py:213-232) */
int pase_bn_prelu_pad_fwd(const void* y, int y_bf16, long y_sample_stride, int N, int T, int C,
                          const float* scale, const float* shift, const float* alpha,
                          void* dst, void* dst_lo, int dst_fmt,
                          long dst_sample_stride, long dst_row_stride,
                          int padL, int padR,
                          float* pool, long pool_sample_stride, long pool_row_stride,
                          int pool_d, int pool_T, void* stream);
/* Packed variable-length form (eval BatchNorm: scale / shift from pase_bn_eval_affine): tab
 * (DEVICE, nseg rows of 6 ints) {T, y_off, dst_off, pool_off, pool_d, pool_T}: utterance i's
 * y[y_off + t*C + c] (t < T) -> dst[dst_off + tau*dst_row_stride + c] with its own reflect halo,
 * and its own dense-skip pool (pool_d, pool_T; pool_T * pool_d <= T) into
 * pool[pool_off + j*pool_row_stride + c] (pool zeroed by the caller; NULL: no pool).  sep != 0
 * also writes zeros to the row ahead of each utterance (dst_off - dst_row_stride, C elements):
 * the x_{t-1} of the QRNN's first step.  max_T >= every T, nseg <= 65535.  One launch for all
 * utterances. */
int pase_bn_prelu_pad_fwd_var(const void* y, int y_bf16, const int* tab, int nseg, int max_T,
                              int C, const float* scale, const float* shift, const float* alpha,
                              void* dst, void* dst_lo, int dst_fmt, long dst_row_stride,
                              int padL, int padR, float* pool, long pool_row_stride, int sep,
                              void* stream);
/* backward, pass 1: g = sum of gradient sources (srcA: fp32 or bf16 as its dgrad GEMM
 * wrote it; srcB / pool: fp32); du = PReLU'(u) g written to dst (same type as y; NULL:
 * not stored, see pase_bn_prelu_bwd_apply_src);
 * accumulates S1=sum du, S2=sum du*xhat, dalpha (double[C] each).  amax (float[2],
 * optional, caller-zeroed): max|du|, max|xhat| for the fp16-pair gradient scale. */
int pase_bn_prelu_bwd_reduce(const void* y, int y_bf16, long y_sample_stride, int N, int T, int C,
                             const float* mean, const float* invstd,
                             const float* scale, const float* shift, const float* alpha,
                             const void* srcA, int a_bf16, long a_sample_stride,
                             long a_row_stride, int padL, int padR,
                             const float* srcB, long b_sample_stride, long b_row_stride,
                             int b_shift,
                             const float* pool, long pool_sample_stride, long pool_row_stride,
                             int pool_d, int pool_T,
                             void* dst, long dst_sample_stride,
                             double* S1, double* S2, double* dalpha, float* amax, void* stream);
/* backward, pass 2: dy = gamma*invstd*(du - S1/M - xhat*S2/M) read from `du` (same type
 * as y; may alias dst when the formats agree) and written as the next GEMMs' operand in
 * format dst_fmt; also finalises db = sum dy.  dst_fmt 2 (fp16 pair): dy is scaled by a
 * power of two s derived from amax (so that it fits fp16) and scale_out = {1/s, s}. */
int pase_bn_prelu_bwd_apply(const void* y, int y_bf16, long y_sample_stride, int N, int T, int C,
                            const float* mean, const float* invstd, const float* gamma,
                            const double* S1, const double* S2, double count,
                            const void* du, void* dst, void* dst_lo, int dst_fmt,
                            long dst_sample_stride, double* dbias_acc,
                            const float* amax, float* scale_out, void* stream);
/* backward of FeBlock's norm -> act (pase/models/modules.py:1072-1075, autograd of
 * BatchNorm1d + PReLU), pass 2 WITHOUT a stored du: du = PReLU'(u) g is recomputed from the gradient
 * sources (arguments as in pass 1, which is then called with dst = NULL and writes only its
 * sums): one write and one read of the layer's activation size less per block. */
int pase_bn_prelu_bwd_apply_src(const void* y, int y_bf16, long y_sample_stride, int N, int T,
                                int C, const float* mean, const float* invstd,
                                const float* gamma, const float* scale, const float* shift,
                                const float* alpha, const double* S1, const double* S2,
                                double count,
                                const void* srcA, int a_bf16, long a_sample_stride,
                                long a_row_stride, int padL, int padR,
                                const float* srcB, long b_sample_stride, long b_row_stride,
                                int b_shift,
                                const float* pool, long pool_sample_stride, long pool_row_stride,
                                int pool_d, int pool_T,
                                void* dst, void* dst_lo, int dst_fmt, long dst_sample_stride,
                                double* dbias_acc, const float* amax, float* scale_out,
                                void* stream);
/* Packed variable-length forms of the two passes above in eval mode (WaveFe.encode_packed,
 * DESIGN.md section 18).  tab (DEVICE, nseg rows of 9 ints) {T, y_off, a_off, b_off, pool_off,
 * pool_d, pool_T, d_off, d_span}: utterance i is a B=1 call with y + y_off, srcA + a_off,
 * srcB + b_off, pool + pool_off (element offsets; the sample strides unused), so its gradient
 * sources are summed as in the uniform kernels.  max_T >= every T.
 * pase_bn_prelu_bwd_reduce_var: pase_bn_prelu_bwd_reduce's sums and maxima over all utterances.
 * pase_bn_prelu_bwd_apply_src_var: pase_bn_prelu_bwd_apply_src with S1 = S2 = 0 (dy = gamma
 * invstd du); utterance i's frame t goes to dst[d_off + t*C ..] (dst rows of C elements), frames
 * T .. d_span-1 after it are written zero and so are the `lead` frames before the first
 * utterance, on every call; max_span >= every d_span.  The fp16-pair scale comes from amax over
 * the whole pack.  dbias_acc (may be NULL) += sum dy. */
int pase_bn_prelu_bwd_reduce_var(const void* y, int y_bf16, const int* tab, int nseg, int max_T,
                                 int C, const float* mean, const float* invstd,
                                 const float* scale, const float* shift, const float* alpha,
                                 const void* srcA, int a_bf16, long a_row_stride, int padL,
                                 int padR, const float* srcB, long b_row_stride, int b_shift,
                                 const float* pool, long pool_row_stride, double* S1, double* S2,
                                 double* dalpha, float* amax, void* stream);
int pase_bn_prelu_bwd_apply_src_var(const void* y, int y_bf16, const int* tab, int nseg,
                                    int max_span, int C, const float* invstd, const float* gamma,
                                    const float* scale, const float* shift, const float* alpha,
                                    const void* srcA, int a_bf16, long a_row_stride, int padL,
                                    int padR, const float* srcB, long b_row_stride, int b_shift,
                                    const float* pool, long pool_row_stride, void* dst,
                                    void* dst_lo, int dst_fmt, int lead, double* dbias_acc,
                                    const float* amax, float* scale_out, void* stream);
/* Train-mode form of pase_bn_prelu_bwd_apply_src_var (WaveFe.encode_packed_train, DESIGN.md
 * section 19; autograd of FeBlock's BatchNorm1d + PReLU over the whole pack,
 * pase/models/modules.py:1014-1077): dy = gamma invstd (du - S1/count - xhat S2/count), xhat =
 * (y - mean) invstd, with S1 = sum du and S2 = sum du xhat of pase_bn_prelu_bwd_reduce_var over
 * every utterance and count = the pack's valid frames.  Table, layout, zero frames, dbias_acc
 * and the fp16-pair scale (bound gamma invstd (max|du| + |S1/count| + max|xhat| |S2/count|)
 * from amax over the pack) as in pase_bn_prelu_bwd_apply_src_var. */
int pase_bn_prelu_bwd_apply_src_var_train(const void* y, int y_bf16, const int* tab, int nseg,
                                          int max_span, int C, const float* mean,
                                          const float* invstd, const float* gamma,
                                          const float* scale, const float* shift,
                                          const float* alpha, const double* S1, const double* S2,
                                          double count, const void* srcA, int a_bf16,
                                          long a_row_stride, int padL, int padR,
                                          const float* srcB, long b_row_stride, int b_shift,
                                          const float* pool, long pool_row_stride, void* dst,
                                          void* dst_lo, int dst_fmt, int lead, double* dbias_acc,
                                          const float* amax, float* scale_out, void* stream);
/* The three backward entry points above read and write y, srcA, srcB, pool, dst, dst_lo and du
 * in quads of channels: fp32 operands must be 16-byte aligned, 16-bit ones 8-byte aligned,
 * every row and sample stride a multiple of 4 elements, a/b_row_stride >= C and
 * pool_T * pool_d <= T; anything else is refused (PASE_ERR_ARG) before a launch.
 * How pass 1 (pase_bn_prelu_bwd_reduce) or pass 2 (pase_bn_prelu_bwd_apply_src; srcA NULL:
 * pase_bn_prelu_bwd_apply with a stored du) runs with these arguments on the current device
 * (host only, launches nothing; arguments as in those calls, dst_lo / dst_fmt only in pass 2):
 * out4 = {path (0: register kernels, 1: staged persistent kernels), time steps per work item
 * (steps per thread or tile rows), work items of all samples (thread runs of one channel
 * quad, or tiles), blocks of the launch (256 threads each)}. */
int pase_bn_bwd_plan(int pass, const void* y, int y_bf16, long y_sample_stride, int N, int T,
                     int C, const void* srcA, int a_bf16, long a_sample_stride,
                     long a_row_stride, int padL, int padR,
                     const float* srcB, long b_sample_stride, long b_row_stride, int b_shift,
                     const float* pool, long pool_sample_stride, long pool_row_stride,
                     int pool_d, int pool_T,
                     void* dst, void* dst_lo, int dst_fmt, long dst_sample_stride, long* out4);
/* plain per-channel PReLU on (rows,C) (MLPBlock / GDeconv1DBlock act) */
int pase_prelu_fwd(const float* u, float* h, const float* alpha, long rows, int C,
                   long ldu, long ldh, void* stream);
int pase_prelu_bwd(const float* u, const float* dh, const float* alpha, float* du,
                   double* dalpha, long rows, int C, long ldu, long lddh, long lddu,
                   void* stream);
/* acc[c] += sum_r X[r*ld+c]  (bias gradients) */
int pase_colsum(const float* X, long ld, long rows, int C, double* acc, void* stream);
int pase_cast_d2f(const double* src, float* dst, int n, float scale, void* stream);

/* ---- output BatchNorm(affine=False) + layout change (frontend.py:206-208,
 * 266-268): (N*T,C) channel-last -> (N,C,T) ------------------------------- */
/* out (N,C,T) = y*scale+shift; optionally also the channel-last copy out_ntc */
int pase_out_affine_nct(const float* y, const float* scale, const float* shift,
                        float* out, float* out_ntc, int N, int T, int C, void* stream);
/* Packed variable-length output with select_output (pase/models/modules.py:62-74) fused:
 * tab (DEVICE, nseg rows of 3 ints) {y_row, T, out_off}; h = y[y_row + t, :]*scale+shift;
 * mode 0: out[out_off..] (C,T) = h; 1 (avg_norm): h - mean_t h; 2 (avg_concat): (2C,T) =
 * [h ; mean_t h]; 3 (avg_norm_concat): [h - mean_t h ; mean_t h].  The time mean is a double
 * sum in a fixed order.  nseg <= 65535. */
int pase_out_affine_var(const float* y, const float* scale, const float* shift, float* out,
                        const int* tab, int nseg, int C, int mode, void* stream);
/* Windowed output of many streams' crops at once (StreamPool, so FeatureStream and
 * WaveFe.extract_long): tab (DEVICE, nseg rows of 5 ints) {row0, T, ocol, ldo, col0}: rows row0
 * .. row0+T-1 of y (rows,C) as y*scale+shift (one fmaf, as pase_out_affine_nct) into columns
 * col0 .. col0+T-1 of the (C, ldo) block starting at element ocol*C of out.  max_T >= every
 * row's T.  64-bit element offsets: the output may exceed 2^31 elements. */
int pase_out_place_var(const float* y, const float* scale, const float* shift, float* out,
                       const int* tab, int nseg, int max_T, int C, void* stream);
/* select_output (pase/models/modules.py:62-74) in place over a whole (C,T) output whose rows
 * 0..C-1 hold h: mode 1 (avg_norm) h - mean_t h; 2 (avg_concat) rows C..2C-1 = mean_t h;
 * 3 (avg_norm_concat) both.  The mean is a double sum in a fixed order. */
int pase_out_select(float* out, long T, int C, int mode, void* stream);
/* g_ntc = dout(N,C,T)^T + dout_ntc; S1 += g, S2 += g*xhat (double[C]) */
int pase_out_bwd_reduce(const float* dout, const float* dout_ntc, const float* y,
                        const float* mean, const float* invstd, int N, int T, int C,
                        float* g_ntc, double* S1, double* S2, void* stream);
/* Packed form of pase_out_bwd_reduce's layout change (eval mode: no statistics): tab (DEVICE,
 * nseg rows of 3 ints) {row0, T, o_off}: g_ntc[(row0 + t)*C + c] = dout[o_off + c*T + t];
 * max_T >= every T. */
int pase_out_bwd_gather_var(const float* dout, const int* tab, int nseg, int max_T, int C,
                            float* g_ntc, void* stream);
/* One window of a recording's backward (WaveFe.encode_long): g_ntc[t*C + c] = dout[c*ld + col0
 * + t - c0] for the crop frames c0 <= t < c0+cn of the window's T frames, 0 for its other frames;
 * dout is the recording's (C, ld) output gradient and col0 (64-bit) its column of frame c0. */
int pase_out_bwd_gather_crop(const float* dout, long ld, long col0, int T, int c0, int cn, int C,
                             float* g_ntc, void* stream);
/* pase_out_bwd_gather_var with pase_out_bwd_reduce's sums (train-mode norm_out of
 * WaveFe.encode_packed_train, frontend.py:206-208): the same gather, and S1 += g,
 * S2 += g*xhat (double[C]) with xhat = (y[(row0 + t)*C + c] - mean[c]) invstd[c] over every
 * utterance's rows; pase_out_bwd_apply(use_stats = 1) then finishes dy. */
int pase_out_bwd_reduce_var(const float* dout, const int* tab, int nseg, int max_T, int C,
                            const float* y, const float* mean, const float* invstd, float* g_ntc,
                            double* S1, double* S2, void* stream);
/* in place: g = scale*(g - use_stats*(S1/M + xhat*S2/M)) */
int pase_out_bwd_apply(float* g, const float* y, const float* mean, const float* invstd,
                       const float* scale, const double* S1, const double* S2,
                       double count, int use_stats, long rows, int C, void* stream);
/* generic (N,C,T) <-> (N,T,C) */
int pase_nct_to_ntc(const float* src, float* dst, int N, int C, int T, long dst_row_stride,
                    void* stream);
int pase_ntc_to_nct(const float* src, long src_row_stride, float* dst, int N, int C, int T,
                    void* stream);

/* ---- QRNN (torchqrnn.QRNN window=2 as called at modules.py:52) ----------- */
/* Y (rows=N*T, 3H) pre-activations -> h (row stride ldh), cell state Cst (rows,H) */
int pase_qrnn_scan_fwd(const float* Y, float* h, long ldh, float* Cst,
                       int N, int T, int H, void* stream);
/* Packed variable-length forward: tab (DEVICE, nseg rows of 2 ints) {row0, T}: rows row0 ..
 * row0+T-1 of Y / h / Cst are one utterance.  Each utterance runs the kernel its own T selects
 * (pase_qrnn_scan_plan), so its result is that of a B=1 scan.  nseg <= 65535.  Two launches. */
int pase_qrnn_scan_fwd_var(const float* Y, float* h, long ldh, float* Cst, const int* tab,
                           int nseg, int H, void* stream);
/* Sequential scans continued over windows of many streams at once (StreamPool, so FeatureStream
 * and WaveFe.extract_long): tab (DEVICE, nseg rows of 4 ints) {row0, T, slot, first}: rows row0
 * .. row0+T-1 of Y / h / Cst continue the scan of the stream whose state is row `slot` of state
 * (max_streams, H), zero when first != 0; the state after the last row is written back there.
 * A slot appears at most once per call.  The per-step arithmetic is the sequential kernel's, so
 * scanning a recording piece by piece reproduces pase_qrnn_scan_fwd's bits for T' > 512. */
int pase_qrnn_scan_fwd_carry_var(const float* Y, float* h, long ldh, float* Cst, float* state,
                                 const int* tab, int nseg, int H, void* stream);
int pase_qrnn_scan_bwd(const float* Y, const float* Cst, const float* dh, long lddh,
                       float* dY, int N, int T, int H, void* stream);
/* Packed variable-length form of pase_qrnn_scan_bwd: tab (DEVICE, nseg rows of 3 ints)
 * {row0, T, drow0}: rows row0 .. row0+T-1 of Y / Cst / dh are one utterance; its gate gradients
 * go to rows drow0 .. drow0+T-1 of dY and row drow0+T of dY is written zero.  Each utterance
 * runs the kernel its own T selects (pase_qrnn_scan_plan), so it gets a B=1 backward's bits.
 * Two launches. */
int pase_qrnn_scan_bwd_var(const float* Y, const float* Cst, const float* dh, long lddh, float* dY,
                           const int* tab, int nseg, int H, void* stream);
/* Backward of pase_qrnn_scan_fwd_carry_var over windows of recordings (WaveFe.encode_long):
 * tab (DEVICE, nseg rows of 6 ints) {row0, T, drow0, c0, cn, slot}: rows row0 .. row0+T-1 of
 * Y / Cst / dh are one window, whose frames c0 .. c0+cn-1 were scanned from row `slot` of state
 * (nslots, H).  Their gate gradients go to rows drow0+c0 .. drow0+c0+cn-1 of dY; rows drow0 ..
 * drow0+T of dY outside them are written zero.  The scan starts from the cell-state gradient in
 * row `slot` of dstate and writes there the gradient of that row of state.  The per-step
 * arithmetic is pase_qrnn_scan_bwd's sequential kernel's.  A slot appears at most once per
 * call. */
int pase_qrnn_scan_bwd_carry_var(const float* Y, const float* Cst, const float* dh, long lddh,
                                 float* dY, const float* state, float* dstate, const int* tab,
                                 int nseg, int H, void* stream);
/* Which kernels the two scans run for T time steps (host only, launches nothing): out1 =
 * segments per block of the time-segmented kernels (16, 24 or 32; T <= 512), or 0 for the
 * sequential kernels (T > 512). */
int pase_qrnn_scan_plan(int T, int* out1);

/* ---- worker losses (losses.py:6-37, utils.py:63-68) ----------------------- */
/* pred (B*T, F*r) channel-last, label (B,F,T): sum (pred - ctx(label))^2 -> acc */
int pase_ctx_mse_fwd(const float* pred, long ldp, const float* label,
                     int B, int F, int T, int r, double* acc, void* stream);
/* dpred = coef * gscale[0] * (pred - ctx(label)) */
int pase_ctx_mse_bwd(const float* pred, long ldp, const float* label,
                     int B, int F, int T, int r, float coef, const float* gscale,
                     float* dpred, long lddp, void* stream);
int pase_l1_fwd(const float* pred, const float* target, long n, double* acc, void* stream);
int pase_l1_bwd(const float* pred, const float* target, long n, float coef,
                const float* gscale, float* dpred, void* stream);
/* BCEWithLogits against labels 1 for rows < half_rows, else 0 */
int pase_bce_pairs_fwd(const float* logit, long n, long n_pos, double* acc, void* stream);
int pase_bce_pairs_bwd(const float* logit, long n, long n_pos, float coef,
                       const float* gscale, float* dlogit, void* stream);
/* time-mean over (B,T,C) channel-last -> (B,C) and its backward (GIM) */
int pase_time_mean_fwd(const float* x, long ldx, float* out, long ldo, int B, int T, int C,
                       void* stream);
int pase_time_mean_bwd(const float* dout, long ldo, float* dx, long ldx, int B, int T, int C,
                       int accumulate, void* stream);
/* SPC frame gather (SPCMinion, minions.py:575-649).  frames: DEVICE int64 {t, future_t, past_t},
 * checked by the host (M + 1 <= t < T - M, t + seq_pad <= future_t < T - N,
 * N <= past_t < t - seq_pad, M = seq_pad + N); the kernels trust them.  x (B*T, C) rows with row
 * stride ldx -> out (2B, (N+1)*C) contiguous: row b = [x(b,t) | fut], row B + b = [x(b,t) | past],
 * fut[c*N + n] = x(b, future_t + n, c), past[c*N + n] = x(b, past_t - N + n, c). */
int pase_spc_gather(const float* x, long ldx, const long* frames, int B, int T, int C, int N,
                    int seq_pad, float* out, void* stream);
/* g (2B, (N+1)*C) -> dense dx (B*T, C): the windows of g copied, g[b, :C] + g[B+b, :C] at frame t,
 * zeros elsewhere (every element written, no atomics). */
int pase_spc_gather_bwd(const float* g, const long* frames, int B, int T, int C, int N,
                        int seq_pad, float* dx, void* stream);
/* ---- StreamPool sample history (csrc/stream.cu) --------------------------- */
/* tab (DEVICE, nrow rows of 8 ints) {slot, head, nnew, stage_off, ring_s, old, seg_len,
 * wave_off}: appends staging[stage_off .. +nnew) to ring slot `slot` (ring + slot*ring_cap,
 * 64-bit) at positions head, head+1, .. mod ring_cap, and writes wave[wave_off .. +seg_len): its
 * first `old` samples from the ring from position ring_s (mod ring_cap), the rest from
 * staging[stage_off + i - old].  The positions read and appended must not overlap.  max_len >=
 * every row's nnew and seg_len.  One launch. */
int pase_stream_gather(const float* staging, float* ring, long ring_cap, float* wave,
                       const int* tab, int nrow, int max_len, void* stream);
/* misc fused vector helpers */
int pase_axpy(const float* x, float* y, long n, float a, void* stream);
int pase_scale_dev(float* x, long n, const float* dev_scalar, float host_coef, void* stream);

/* ---- optimizer (SURVEY 8f N4): the reference steps 13 torch.optim.Adam or RAdam instances
 * (trainer.py:86-143, worker_scheduler.py:66-73); here ONE launch updates every
 * parameter of the flat fp32 buffers.  seg_table: device array of nseg rows of 6 x 8
 * bytes {long start, long end, float lr, float beta1, float beta2, float eps,
 * float weight_decay, float algorithm, long step_index}; segments are sorted, disjoint and
 * start at multiples of 4 elements; steps: device float vector of step counts (already
 * incremented for this update).  grad_scale multiplies the gradient (1/world of a
 * summed all-reduce, or 1).  algorithm 0: torch.optim.Adam (amsgrad / maximize off, L2
 * weight decay); 1: the reference's RAdam (WorkerScheduler/radam.py: rho and the step size
 * in fp64 from the step count, momentum-SGD step while rho < 5, decoupled weight decay). */
int pase_adam_flat(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long n,
                   const long* seg_table, int nseg, const float* steps, float grad_scale,
                   void* stream);
/* Data parallelism fused into the update (the reference is single-GPU: its per-worker
 * optimizer instances, trainer.py:86-143 / worker_scheduler.py:66-73, have no exchange step; this
 * replaces ncclAllReduce + the update above, see SURVEY.md 8e): every rank's flat gradient / parameter / flag buffers are peer-mapped
 * (param_peers / grad_peers / flag_peers: DEVICE arrays of `world` pointers; flags: int[2*world]
 * per rank, zero-initialised).  One launch per rank and step: cross-GPU barrier, mean of the
 * peers' gradients over this rank's 1/world shard read through NVLink, each segment's update
 * (the same arithmetic as pase_adam_flat) on the local
 * (exp_avg, exp_avg_sq) shard, new parameters stored into every rank's buffer, barrier.
 * epoch / done: zero-initialised device scalars owned by the optimizer.  n % 4 == 0. */
int pase_adam_flat_dp(void* const* param_peers, void* const* grad_peers,
                      void* const* flag_peers, float* exp_avg, float* exp_avg_sq, long n,
                      const long* seg_table, int nseg, const float* steps, int world, int rank,
                      int* epoch, int* done, void* stream);
/* peer-mapped buffers for pase_adam_flat_dp (CUDA IPC; same node, one process per GPU):
 * alloc: zeroed cudaMalloc buffer on the current device + its 64-byte IPC handle;
 * open: map a peer's buffer (handle received out of band) into the current device's address
 * space with peer access; close / free: the inverse operations. */
int pase_dp_alloc(long bytes, void** ptr_out, void* handle_out64);
int pase_dp_open(const void* handle64, void** ptr_out);
int pase_dp_close(void* ptr);
int pase_dp_free(void* ptr);

/* ---- on-device regression targets (pase/transforms.py:439-487 LPS, 183-202 ZNorm) ---- */
/* frames matrix of the STFT as an fp16 (hi, lo') pair GEMM operand: row (n, j), column m =
 * x[n][reflect(j*hop + start0 + m)] for m < win (the samples the rectangular window keeps;
 * start0 = (n_fft - win)/2 - n_fft/2), zero for win <= m < lda. */
int pase_frame_wave(const float* x, int N, int T, int hop, int win, int start0, int frames,
                    void* hi, void* lo, int lda, void* stream);
/* C (N*frames, ldc): columns (2k, 2k+1) = (re, im) of bin k.  out (N, (1+der_order)*nbins,
 * frames): 10 log10(|X|^2 + 1e-19), then its Savitzky-Golay derivatives of order 1..der_order
 * along time (fir: der_order rows of `width` correlation taps; edge frames use the nearest
 * full window = scipy/librosa mode 'interp' with polyorder == deriv), optionally
 * (v - mean[f]) / std[f] per feature row. */
int pase_lps_post(const float* C, long ldc, int N, int frames, int nbins, int der_order,
                  int width, const float* fir, const float* mean, const float* stdv, float* out,
                  void* stream);

/* ---- on-device waveform distortions (pase/transforms.py:38-146 config_distortions /
 * PCompose; the host planner is pase_b200/distortions.py).  Job tables are int64 DEVICE rows,
 * one per sample (row b acts on row b of every operand); a row whose first field is 0 is not
 * drawn and its sample is left untouched, and a row that does not fit its operands is treated
 * the same way.  Rows of x / out / seg / label are `ld*` elements apart.  Reductions are fp64
 * in a fixed order, so results are reproducible bit for bit. */
/* Workspace bytes pase_fft_conv needs for this geometry (host-only). */
int pase_fft_conv_workspace(int njobs, int T, int Lmax, long* bytes);
/* FFT convolution + energy scale (Reverb transforms.py:1071-1103, BandDrop 1263-1297,
 * Downsample 1162-1197).  jobs: njobs rows {on, n, filt_off, L, p, mode}, n <= T, L <= Lmax,
 * 0 <= p < L, filt_off + L <= bank_len.  With h = bank[filt_off, +L) and
 * full = signal.convolve(x[0, n), h, 'full'), y[t] = full[p + t] for t < n:
 *   mode 0 (FIR):    E = y.y;    out = sqrt(Ex/E) y if E > 0, else x
 *   mode 1 (reverb): E = full.full (tail included); out = sqrt(Ex/E) y if E > 0, else y
 *   mode 2 (raw):    out = y
 * where Ex = x[0,n).x[0,n).  out may equal x (in place); out[n, T) is not written.  Uniformly
 * partitioned overlap-save: 4096-sample blocks, 8192-point fp32 FFTs in shared memory.
 * twiddle: 4096 (re, im) pairs exp(-2 pi i k / 8192).  ws: >= pase_fft_conv_workspace bytes,
 * 16-byte aligned. */
int pase_fft_conv(const float* x, long ldx, const float* bank, long bank_len, const long* jobs,
                  int njobs, int T, int Lmax, const float* twiddle, void* ws, long ws_bytes,
                  float* out, long ldo, void* stream);
/* Noise / overlap segment (transforms.py:1644-1658, 1720-1733): jobs rows {on, pool_off,
 * avail}; out[u] = pool[pool_off + u] for u < avail, 0 for avail <= u < T. */
int pase_segment_gather(const float* pool, long pool_len, const long* jobs, int njobs, int T,
                        float* out, long ldo, void* stream);
/* In-place additive mix (SimpleAdditive transforms.py:1633-1675 with guard = 1,
 * SimpleAdditiveShift 1714-1766 with guard = 0): jobs rows {on, shift, guard}; the noise is
 * n[t] = 0 for t < shift, seg[t - shift] after; K = sqrt(Ex / (snr_lin En)) (1 if En == 0);
 * x <- sqrt(Ex / (v.v + 1e-14)) v with v = x + K n.  guard: En == 0 leaves x as it is. */
int pase_noise_mix(float* x, long ldx, const float* seg, long lds, const long* jobs,
                   const double* snr_lin, int njobs, int T, void* stream);
/* In-place Clipping (transforms.py:1522-1536): jobs rows {on};
 * x <- min(max(x, cf min x), cf max x). */
int pase_clip(float* x, long ldx, const long* jobs, const double* cf, int njobs, int T,
              void* stream);
/* Overlap label (transforms.py:1738-1748): jobs rows {on, shift, guard} (the overlap mix
 * table); label[j] = mean of (t >= shift) over t in [j d, (j+1) d), 0 where on == 0.
 * d divides T. */
int pase_overlap_label(const long* jobs, int njobs, int T, int d, float* label, long ldl,
                       void* stream);

/* ---- on-device batch assembly (pase/dataset.py:452-513 LibriSpeechSegTupleWavDataset,
 * pase/transforms.py:295-436 SingleChunkWav / MIChunkWav, 253-292 CachedCompose; the host
 * planner is pase_b200/batch.py).  Row tables are int64 DEVICE rows drawn and bounds-checked
 * by the planner; a row that does not fit its pool is skipped (its output is not written).
 * Pools may be device memory or page-locked host memory read through its mapped address. */
/* Chunk windows: rows (B, nsrc, 6) {fmt, off, L, beg, scale, rbits}; CTA (s, b) reads
 * x[j] = u[beg + j], j < T, of utterance u = pool[off, off + L) (fmt 0: pcm int16 k / 32768,
 * fmt 1: flt fp32), reflected past its end (u[L + i] = u[L - 2 - i]).  scale != 0:
 * x <- __fmul_rn(__fdiv_rn(x, max|x|), r), r = the fp32 with bits rbits (a silent window gives
 * 0/0 = NaN, as the reference's norm_and_scale).  Writes out[s * plane + b * T + j] and, for
 * s == 0 when cchunk != 0, the copy at out[nsrc * plane + b * T + j]. */
int pase_chunk_gather(const void* pcm, long pcm_len, const float* flt, long flt_len,
                      const long* rows, int B, int nsrc, int T, int cchunk, float* out,
                      long plane, void* stream);
/* Cached-feature slices: rows (B, 3) {off, frames, s}; out (B, F, n) with
 * out[b, f, t] = pool[off + f * frames + s + t], s + n <= frames. */
int pase_frames_gather(const float* pool, long pool_len, const long* rows, int B, int F, int n,
                       float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
