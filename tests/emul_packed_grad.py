"""TEST-ONLY torch emulation of the packed backward entry points (include/pase_b200.h,
pase_*_var of WaveFe.encode_packed): each utterance of a table is run through the emulation of
the uniform entry point it generalises (tests/emul_ops.py, tests/emul_input_grad.py); the
forward's packed entry points come from tests/emul_extract.py."""
import torch

import emul_extract
import emul_input_grad
import emul_ops

_ROW = 9


def _rows(tab, n, width):
    return tab[:n * width].view(n, width).tolist()


def pase_bn_prelu_bwd_reduce_var(y, y_bf16, tab, nseg, max_T, C, mean, invstd, scale, shift,
                                 alpha, A, a_bf16, a_rs, padL, padR, B, b_rs, b_shift, pool,
                                 p_rs, S1, S2, dalpha, amax):
    for T, y_off, a_off, b_off, p_off, pool_d, pool_T, _, _ in _rows(tab, nseg, _ROW):
        assert T <= max_T
        emul_ops.pase_bn_prelu_bwd_reduce(
            y[y_off:], y_bf16, 0, 1, T, C, mean, invstd, scale, shift, alpha, A[a_off:], a_bf16,
            0, a_rs, padL, padR, None if B is None else B[b_off:], 0, b_rs, b_shift,
            None if pool is None else pool[p_off:], 0, p_rs, pool_d if pool is not None else 0,
            pool_T, None, 0, S1, S2, dalpha, amax)


def pase_bn_prelu_bwd_apply_src_var(y, y_bf16, tab, nseg, max_span, C, invstd, gamma, scale,
                                    shift, alpha, A, a_bf16, a_rs, padL, padR, B, b_rs, b_shift,
                                    pool, p_rs, dst, dst_lo, dst_fmt, lead, dbias, amax,
                                    scale_out):
    zeros = torch.zeros(2 * C, dtype=torch.float64)
    for i, (T, y_off, a_off, b_off, p_off, pool_d, pool_T, d_off, span) in \
            enumerate(_rows(tab, nseg, _ROW)):
        assert T <= span <= max_span
        emul_ops.pase_bn_prelu_bwd_apply_src(
            y[y_off:], y_bf16, 0, 1, T, C, torch.zeros(C), invstd, gamma, scale, shift, alpha,
            zeros[:C], zeros[C:], 1.0, A[a_off:], a_bf16, 0, a_rs, padL, padR,
            None if B is None else B[b_off:], 0, b_rs, b_shift,
            None if pool is None else pool[p_off:], 0, p_rs, pool_d if pool is not None else 0,
            pool_T, dst[d_off:], None if dst_lo is None else dst_lo[d_off:], dst_fmt, 0, dbias,
            amax, scale_out)
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


def pase_qrnn_scan_bwd_var(Y, Cst, dh, lddh, dY, tab, nseg, H):
    for row0, T, drow0 in _rows(tab, nseg, 3):
        emul_ops.pase_qrnn_scan_bwd(Y[row0 * 3 * H:], Cst[row0 * H:], dh[row0 * lddh:], lddh,
                                    dY[drow0 * 3 * H:], 1, T, H)
        dY[(drow0 + T) * 3 * H:(drow0 + T + 1) * 3 * H] = 0


def pase_reflect_fold_wave_var(dpad, tab, nseg, max_T, dx, padL, padR):
    for x_off, T, d_off in _rows(tab, nseg, 3):
        assert T <= max_T
        emul_input_grad.pase_reflect_fold_wave(dpad[d_off:], T + padL + padR, dx[x_off:], 1, T,
                                               padL, padR)


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        if hasattr(emul_input_grad, name):
            return emul_input_grad.call(name, *args)
        return emul_extract.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
