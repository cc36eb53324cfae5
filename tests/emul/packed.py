"""The packed variable-length entry points (pase_*_var of WaveFe.encode_packed and
encode_packed_train): each utterance of a table runs through the emulation of the uniform entry
point it generalises, train-mode statistics accumulated over the whole pack."""
import torch

from pase_b200.modules import select_output

from . import core, input_grad
from .core import _MODES, _rows

_ROW = 9      # columns of the BatchNorm/PReLU backward tables


def _var_map(tab, n):
    t = tab[:3 * n + 1].tolist()
    return [(t[i], t[i + 1] - t[i], t[n + 1 + i], t[2 * n + 1 + i]) for i in range(n)]


# ---- forward
def pase_reflect_pad_wave_var(x, tab, nseg, max_T, dst, dst_lo, dst_fmt, padL, padR):
    for x_off, T, d_off in _rows(tab, nseg, 3):
        assert T <= max_T
        core.pase_reflect_pad_wave(x[x_off:], dst[d_off:],
                                   None if dst_lo is None else dst_lo[d_off:], dst_fmt, 1, T,
                                   padL, padR, T + padL + padR)


def pase_bn_prelu_pad_fwd_var(y, y_bf16, tab, nseg, max_T, C, scale, shift, alpha, dst, dst_lo,
                              dst_fmt, d_rs, padL, padR, pool, p_rs, sep):
    for T, y_off, d_off, p_off, pool_d, pool_T in _rows(tab, nseg, 6):
        assert T <= max_T
        if sep:
            dst[d_off - d_rs:d_off - d_rs + C] = 0
            if dst_lo is not None:
                dst_lo[d_off - d_rs:d_off - d_rs + C] = 0
        core.pase_bn_prelu_pad_fwd(
            y[y_off:], y_bf16, 0, 1, T, C, scale, shift, alpha, dst[d_off:],
            None if dst_lo is None else dst_lo[d_off:], dst_fmt, 0, d_rs, padL, padR,
            None if pool is None else pool[p_off:], 0, p_rs, pool_d if pool is not None else 0,
            pool_T)


def pase_gemm_nt_var(A, lda, B, ldb, C, ldc, M, N, K, bias, tab, nvar, fold):
    pase_gemm_nt_var_stats(A, lda, B, ldb, C, ldc, M, N, K, bias, tab, nvar, fold, None, None)


def pase_gemm_nt_var_stats(A, lda, B, ldb, C, ldc, M, N, K, bias, tab, nvar, fold, colsum,
                           colsumsq):
    for r0, P, o0, tv in _var_map(tab, nvar):
        assert r0 + P <= M
        core.pase_gemm_nt(A[r0 * lda:], lda, B, ldb, C[o0 * ldc:], ldc, P, N, K, 1.0, bias,
                          P, tv, P, fold, colsum, colsumsq, 0)


def pase_tc_gemm_nt_var(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, bias, tab, nvar,
                        fold, mode, c_bf16):
    pase_tc_gemm_nt_var_stats(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, bias, tab,
                              nvar, fold, None, None, mode, c_bf16)


def pase_tc_gemm_nt_var_stats(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, bias, tab,
                              nvar, fold, colsum, colsumsq, mode, c_bf16):
    for r0, P, o0, tv in _var_map(tab, nvar):
        assert r0 + P <= M
        core.pase_tc_gemm_nt(Ahi[r0 * R:], None if Alo is None else Alo[r0 * R:], a_rows - r0,
                             R, Bhi, Blo, ldb, C[o0 * ldc:], ldc, P, N, K, 1.0, None, bias,
                             P, tv, P, fold, colsum, colsumsq, 0, mode, c_bf16)


def pase_qrnn_scan_fwd_var(Y, h, ldh, Cst, tab, nseg, H):
    for r0, T in _rows(tab, nseg, 2):
        core.pase_qrnn_scan_fwd(Y[r0 * 3 * H:], h[r0 * ldh:], ldh, Cst[r0 * H:], 1, T, H)


def pase_out_affine_var(y, scale, shift, out, tab, nseg, C, mode):
    for r0, T, o in _rows(tab, nseg, 3):
        v = (y[r0 * C:(r0 + T) * C].view(T, C).double() * scale[:C].double()
             + shift[:C].double()).float()
        f = select_output(v.t().contiguous().view(1, C, T), _MODES[mode])
        out[o:o + f.numel()] = f.reshape(-1)


# ---- backward
def pase_bn_prelu_bwd_reduce_var(y, y_bf16, tab, nseg, max_T, C, mean, invstd, scale, shift,
                                 alpha, A, a_bf16, a_rs, padL, padR, B, b_rs, b_shift, pool,
                                 p_rs, S1, S2, dalpha, amax):
    for T, y_off, a_off, b_off, p_off, pool_d, pool_T, _, _ in _rows(tab, nseg, _ROW):
        assert T <= max_T
        core.pase_bn_prelu_bwd_reduce(
            y[y_off:], y_bf16, 0, 1, T, C, mean, invstd, scale, shift, alpha, A[a_off:], a_bf16,
            0, a_rs, padL, padR, None if B is None else B[b_off:], 0, b_rs, b_shift,
            None if pool is None else pool[p_off:], 0, p_rs, pool_d if pool is not None else 0,
            pool_T, None, 0, S1, S2, dalpha, amax)


def pase_bn_prelu_bwd_apply_src_var(y, y_bf16, tab, nseg, max_span, C, invstd, gamma, scale,
                                    shift, alpha, A, a_bf16, a_rs, padL, padR, B, b_rs, b_shift,
                                    pool, p_rs, dst, dst_lo, dst_fmt, lead, dbias, amax,
                                    scale_out):
    """Eval-mode BatchNorm: the train-mode form with zero batch statistics."""
    zeros = torch.zeros(2 * C, dtype=torch.float64)
    pase_bn_prelu_bwd_apply_src_var_train(
        y, y_bf16, tab, nseg, max_span, C, torch.zeros(C), invstd, gamma, scale, shift, alpha,
        zeros[:C], zeros[C:], 1.0, A, a_bf16, a_rs, padL, padR, B, b_rs, b_shift, pool, p_rs,
        dst, dst_lo, dst_fmt, lead, dbias, amax, scale_out)


def pase_bn_prelu_bwd_apply_src_var_train(y, y_bf16, tab, nseg, max_span, C, mean, invstd, gamma,
                                          scale, shift, alpha, S1, S2, count, A, a_bf16, a_rs,
                                          padL, padR, B, b_rs, b_shift, pool, p_rs, dst, dst_lo,
                                          dst_fmt, lead, dbias, amax, scale_out):
    for i, (T, y_off, a_off, b_off, p_off, pool_d, pool_T, d_off, span) in \
            enumerate(_rows(tab, nseg, _ROW)):
        assert T <= span <= max_span
        core.pase_bn_prelu_bwd_apply_src(
            y[y_off:], y_bf16, 0, 1, T, C, mean, invstd, gamma, scale, shift, alpha, S1, S2,
            count, A[a_off:], a_bf16, 0, a_rs, padL, padR, None if B is None else B[b_off:], 0,
            b_rs, b_shift, None if pool is None else pool[p_off:], 0, p_rs,
            pool_d if pool is not None else 0, pool_T, dst[d_off:],
            None if dst_lo is None else dst_lo[d_off:], dst_fmt, 0, dbias, amax, scale_out)
        spans = [(d_off + T * C, d_off + span * C)]
        if i == 0:
            spans.append((d_off - lead * C, d_off))
        for a, b in spans:
            dst[a:b] = 0
            if dst_lo is not None:
                dst_lo[a:b] = 0


def pase_out_bwd_gather_var(dout, tab, nseg, max_T, C, g):
    for row0, T, o in _rows(tab, nseg, 3):
        assert T <= max_T
        g[row0 * C:(row0 + T) * C] = dout[o:o + C * T].view(C, T).t().reshape(-1)


def pase_out_bwd_reduce_var(dout, tab, nseg, max_T, C, y, mean, invstd, g, S1, S2):
    for row0, T, o in _rows(tab, nseg, 3):
        assert T <= max_T
        core.pase_out_bwd_reduce(dout[o:], None, y[row0 * C:], mean, invstd, 1, T, C,
                                 g[row0 * C:], S1, S2)


def pase_qrnn_scan_bwd_var(Y, Cst, dh, lddh, dY, tab, nseg, H):
    for row0, T, drow0 in _rows(tab, nseg, 3):
        core.pase_qrnn_scan_bwd(Y[row0 * 3 * H:], Cst[row0 * H:], dh[row0 * lddh:], lddh,
                                dY[drow0 * 3 * H:], 1, T, H)
        dY[(drow0 + T) * 3 * H:(drow0 + T + 1) * 3 * H] = 0


def pase_reflect_fold_wave_var(dpad, tab, nseg, max_T, dx, padL, padR):
    for x_off, T, d_off in _rows(tab, nseg, 3):
        assert T <= max_T
        input_grad.pase_reflect_fold_wave(dpad[d_off:], T + padL + padR, dx[x_off:], 1, T,
                                          padL, padR)
