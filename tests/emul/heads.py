"""The worker-head entry points of the SPC frame gather (pase_b200/csrc/spc.cu) and the fused
contextual-MSE GEMM of the regression heads."""
import torch

from .core import F16_LO_MUL, _as, _ctx, _operand


def _windows(frames, N):
    t, ft, pt = [int(v) for v in frames.tolist()]
    return t, ft, pt - N


def pase_spc_gather(x, ldx, frames, B, T, C, N, seq_pad, out):
    t, ft, p0 = _windows(frames, N)
    v = torch.as_strided(x, (B, T, C), (T * ldx, ldx, 1), x.storage_offset())
    cur = v[:, t]
    fut = v[:, ft:ft + N].transpose(1, 2).reshape(B, -1)        # index c * N + n
    past = v[:, p0:p0 + N].transpose(1, 2).reshape(B, -1)
    out.view(2 * B, -1).copy_(torch.cat([torch.cat([cur, fut], 1), torch.cat([cur, past], 1)], 0))


def pase_spc_gather_bwd(g, frames, B, T, C, N, seq_pad, dx):
    t, ft, p0 = _windows(frames, N)
    G = g.reshape(2 * B, (N + 1) * C)
    d = dx.view(B, T, C)
    d.zero_()
    gf = G[:B, C:].reshape(B, C, N)
    gp = G[B:, C:].reshape(B, C, N)
    d[:, ft:ft + N] = gf.transpose(1, 2)
    d[:, p0:p0 + N] = gp.transpose(1, 2)
    cur = G[:B, :C] + G[B:, :C]
    d[:, t] = cur + gf[:, :, t - ft] if ft <= t < ft + N else cur


def pase_tc_gemm_nt_ctxmse(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, Rhi, Rlo, ldr, M, N, K, bias, label,
                           B, F, T, r, scale, loss_acc, db_acc):
    """loss_acc += sum residual^2, residual[m, n] = sum_k A[m,k] B[n,k] + bias[n] -
    label[b][n/r][t + n%r - r/2]; db_acc += the column sums of the residual, and Rhi / Rlo get
    it as an fp16 pair scaled by scale[1].  Rhi, Rlo and db_acc all None: the loss-only form,
    which writes loss_acc alone."""
    loss_only = Rhi is None
    assert not loss_only or (Rlo is None and db_acc is None), \
        "loss only: Rhi, Rlo and db_acc all NULL"
    assert M == B * T and N == F * r and ldr % 128 == 0 and (not loss_only or ldr >= N)
    need = M * R + K
    A = torch.zeros(need)
    lim = min(a_rows * R, Ahi.numel(), need)
    A[:lim] = _operand(Ahi, Alo, 3, lim)
    Bm = _operand(Bhi, Blo, 3, N * ldb)
    a = _as(A, (M, K), (R, 1)).double()
    b = _as(Bm, (N, K), (ldb, 1)).double()
    pred = a @ b.t()
    if bias is not None:
        pred = pred + bias[:N].double()[None, :]
    d = (pred - _ctx(label, B, F, T, r).double())
    loss_acc[0] += (d * d).sum()
    if loss_only:
        return
    db_acc[:N] += d.sum(0)
    s = float(scale[1])
    v = (d * s).float()
    hi = v.to(torch.float16)
    out_hi = torch.zeros(M, ldr, dtype=torch.float16)
    out_lo = torch.zeros(M, ldr, dtype=torch.float16)
    out_hi[:, :N] = hi
    out_lo[:, :N] = ((v - hi.float()) * F16_LO_MUL).to(torch.float16)
    Rhi[:M * ldr] = out_hi.reshape(-1)
    Rlo[:M * ldr] = out_lo.reshape(-1)
