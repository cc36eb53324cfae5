"""TEST-ONLY torch emulation of the packed variable-length entry points (include/pase_b200.h,
*_var): each utterance of a table is run through the emulation of the uniform entry point it
generalises (tests/emul_ops.py), so the packed forward can be checked on a GPU-less box."""
import torch

import emul_ops
from pase_b200.modules import select_output

_MODES = {0: None, 1: "avg_norm", 2: "avg_concat", 3: "avg_norm_concat"}


def _rows(tab, n, width):
    return tab[:n * width].view(n, width).tolist()


def _var_map(tab, n):
    t = tab[:3 * n + 1].tolist()
    return [(t[i], t[i + 1] - t[i], t[n + 1 + i], t[2 * n + 1 + i]) for i in range(n)]


def pase_reflect_pad_wave_var(x, tab, nseg, max_T, dst, dst_lo, dst_fmt, padL, padR):
    for x_off, T, d_off in _rows(tab, nseg, 3):
        assert T <= max_T
        emul_ops.pase_reflect_pad_wave(x[x_off:], dst[d_off:],
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
        emul_ops.pase_bn_prelu_pad_fwd(
            y[y_off:], y_bf16, 0, 1, T, C, scale, shift, alpha, dst[d_off:],
            None if dst_lo is None else dst_lo[d_off:], dst_fmt, 0, d_rs, padL, padR,
            None if pool is None else pool[p_off:], 0, p_rs, pool_d if pool is not None else 0,
            pool_T)


def pase_gemm_nt_var(A, lda, B, ldb, C, ldc, M, N, K, bias, tab, nvar, fold):
    for r0, P, o0, tv in _var_map(tab, nvar):
        assert r0 + P <= M
        emul_ops.pase_gemm_nt(A[r0 * lda:], lda, B, ldb, C[o0 * ldc:], ldc, P, N, K, 1.0, bias,
                              P, tv, P, fold, None, None, 0)


def pase_tc_gemm_nt_var(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, bias, tab, nvar,
                        fold, mode, c_bf16):
    for r0, P, o0, tv in _var_map(tab, nvar):
        assert r0 + P <= M
        emul_ops.pase_tc_gemm_nt(Ahi[r0 * R:], None if Alo is None else Alo[r0 * R:], a_rows - r0,
                                 R, Bhi, Blo, ldb, C[o0 * ldc:], ldc, P, N, K, 1.0, None, bias,
                                 P, tv, P, fold, None, None, 0, mode, c_bf16)


def pase_qrnn_scan_fwd_var(Y, h, ldh, Cst, tab, nseg, H):
    for r0, T in _rows(tab, nseg, 2):
        emul_ops.pase_qrnn_scan_fwd(Y[r0 * 3 * H:], h[r0 * ldh:], ldh, Cst[r0 * H:], 1, T, H)


def pase_out_affine_var(y, scale, shift, out, tab, nseg, C, mode):
    for r0, T, o in _rows(tab, nseg, 3):
        v = (y[r0 * C:(r0 + T) * C].view(T, C).double() * scale[:C].double()
             + shift[:C].double()).float()
        f = select_output(v.t().contiguous().view(1, C, T), _MODES[mode])
        out[o:o + f.numel()] = f.reshape(-1)


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        return emul_ops.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
