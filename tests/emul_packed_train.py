"""TEST-ONLY torch emulation of the train-mode packed entry points (include/pase_b200.h, the
entry points of WaveFe.encode_packed_train): each utterance of a table is run through the
emulation of the uniform entry point it generalises (tests/emul_ops.py), with the statistics
accumulated over the whole pack; every other packed entry point comes from
tests/emul_packed_grad.py."""
import torch

import emul_extract
import emul_ops
import emul_packed_grad

_ROW = 9


def pase_gemm_nt_var_stats(A, lda, B, ldb, C, ldc, M, N, K, bias, tab, nvar, fold, colsum,
                           colsumsq):
    for r0, P, o0, tv in emul_extract._var_map(tab, nvar):
        assert r0 + P <= M
        emul_ops.pase_gemm_nt(A[r0 * lda:], lda, B, ldb, C[o0 * ldc:], ldc, P, N, K, 1.0, bias,
                              P, tv, P, fold, colsum, colsumsq, 0)


def pase_tc_gemm_nt_var_stats(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, bias, tab,
                              nvar, fold, colsum, colsumsq, mode, c_bf16):
    for r0, P, o0, tv in emul_extract._var_map(tab, nvar):
        assert r0 + P <= M
        emul_ops.pase_tc_gemm_nt(Ahi[r0 * R:], None if Alo is None else Alo[r0 * R:], a_rows - r0,
                                 R, Bhi, Blo, ldb, C[o0 * ldc:], ldc, P, N, K, 1.0, None, bias,
                                 P, tv, P, fold, colsum, colsumsq, 0, mode, c_bf16)


def pase_bn_prelu_bwd_apply_src_var_train(y, y_bf16, tab, nseg, max_span, C, mean, invstd, gamma,
                                          scale, shift, alpha, S1, S2, count, A, a_bf16, a_rs,
                                          padL, padR, B, b_rs, b_shift, pool, p_rs, dst, dst_lo,
                                          dst_fmt, lead, dbias, amax, scale_out):
    for i, (T, y_off, a_off, b_off, p_off, pool_d, pool_T, d_off, span) in \
            enumerate(emul_packed_grad._rows(tab, nseg, _ROW)):
        assert T <= span <= max_span
        emul_ops.pase_bn_prelu_bwd_apply_src(
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


def pase_out_bwd_reduce_var(dout, tab, nseg, max_T, C, y, mean, invstd, g, S1, S2):
    for row0, T, o in emul_packed_grad._rows(tab, nseg, 3):
        assert T <= max_T
        emul_ops.pase_out_bwd_reduce(dout[o:], None, y[row0 * C:], mean, invstd, 1, T, C,
                                     g[row0 * C:], S1, S2)


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        return emul_packed_grad.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
