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
int pase_tc_gemm_tn(const void* Ahi, const void* Alo, long lda, int pitchA, int offA,
                    const void* Bhi, const void* Blo, int R, int pitchB, long b_rows_total,
                    float* C, long ldc, int I, int J, int groups, int rows_per_group,
                    float alpha, const float* alpha_dev, int accumulate, int mode, void* stream);

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
 * scale = device {1/s, s} (pase_bound_scale of the Cauchy-Schwarz bound). */
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
/* g_ntc = dout(N,C,T)^T + dout_ntc; S1 += g, S2 += g*xhat (double[C]) */
int pase_out_bwd_reduce(const float* dout, const float* dout_ntc, const float* y,
                        const float* mean, const float* invstd, int N, int T, int C,
                        float* g_ntc, double* S1, double* S2, void* stream);
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
int pase_qrnn_scan_bwd(const float* Y, const float* Cst, const float* dh, long lddh,
                       float* dY, int N, int T, int H, void* stream);

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
/* misc fused vector helpers */
int pase_axpy(const float* x, float* y, long n, float a, void* stream);
int pase_scale_dev(float* x, long n, const float* dev_scalar, float host_coef, void* stream);

/* ---- optimizer (SURVEY 8f N4): the reference steps 13 torch.optim.Adam instances
 * (trainer.py:86-143, worker_scheduler.py:66-73); here ONE launch updates every
 * parameter of the flat fp32 buffers.  seg_table: device array of nseg rows of 6 x 8
 * bytes {long start, long end, float lr, float beta1, float beta2, float eps,
 * float weight_decay, float pad, long step_index}; segments are sorted, disjoint and
 * start at multiples of 4 elements; steps: device float vector of step counts (already
 * incremented for this update).  grad_scale multiplies the gradient (1/world of a
 * summed all-reduce, or 1).  Semantics = torch.optim.Adam (amsgrad / maximize off). */
int pase_adam_flat(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long n,
                   const long* seg_table, int nseg, const float* steps, float grad_scale,
                   void* stream);
/* Data parallelism fused into the update (the reference is single-GPU: its per-worker Adam
 * instances, trainer.py:86-143 / worker_scheduler.py:66-73, have no exchange step; this
 * replaces ncclAllReduce + the update above, see SURVEY.md 8e): every rank's flat gradient / parameter / flag buffers are peer-mapped
 * (param_peers / grad_peers / flag_peers: DEVICE arrays of `world` pointers; flags: int[2*world]
 * per rank, zero-initialised).  One launch per rank and step: cross-GPU barrier, mean of the
 * peers' gradients over this rank's 1/world shard read through NVLink, Adam on the local
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

#ifdef __cplusplus
}
#endif
#endif
