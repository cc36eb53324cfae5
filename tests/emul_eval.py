"""TEST-ONLY emulation of the loss-only form of pase_tc_gemm_nt_ctxmse (include/pase_b200.h:
Rhi, Rlo and db_acc all NULL) with torch CPU operations.  ``call`` replaces
``pase_b200.ops.call``: the full form and every other entry point go to emul_spc / emul_ops, so
the validation pass can be checked on a GPU-less box.  Never imported by the product.
"""
import torch

import emul_ops
import emul_spc


def ctxmse_loss_only(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, ldr, M, N, K, bias, label, B, F, T, r,
                     loss_acc):
    """loss_acc += sum residual^2, residual[m, n] = sum_k A[m,k] B[n,k] + bias[n] -
    label[b][n/r][t + n%r - r/2]; nothing else is written."""
    assert M == B * T and N == F * r and ldr % 128 == 0 and ldr >= N
    need = M * R + K
    A = torch.zeros(need)
    lim = min(a_rows * R, Ahi.numel(), need)
    A[:lim] = emul_ops._operand(Ahi, Alo, 3, lim)
    Bm = emul_ops._operand(Bhi, Blo, 3, N * ldb)
    a = emul_ops._as(A, (M, K), (R, 1)).double()
    b = emul_ops._as(Bm, (N, K), (ldb, 1)).double()
    pred = a @ b.t()
    if bias is not None:
        pred = pred + bias[:N].double()[None, :]
    d = pred - emul_ops._ctx(label, B, F, T, r).double()
    loss_acc[0] += (d * d).sum()


def call(name, *args):
    if name == "pase_tc_gemm_nt_ctxmse" and args[7] is None:
        (Ahi, Alo, a_rows, R, Bhi, Blo, ldb, Rhi, Rlo, ldr, M, N, K, bias, label, B, F, T, r,
         scale, loss_acc, db_acc) = args
        assert Rlo is None and db_acc is None, "loss only: Rhi, Rlo and db_acc all NULL"
        with torch.no_grad():
            ctxmse_loss_only(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, ldr, M, N, K, bias, label, B,
                             F, T, r, loss_acc)
        return 0
    return emul_spc.call(name, *args)
