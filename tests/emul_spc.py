"""TEST-ONLY emulation of the SPC frame-gather entry points of include/pase_b200.h
(pase_b200/csrc/spc.cu) with torch CPU operations.  ``call`` replaces ``pase_b200.ops.call``
(delegating every other entry point to emul_ops) so that SPCMinion's host path and the training
step planner can be checked on a GPU-less box.  Never imported by the product.
"""
import torch

import emul_ops


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


def call(name, *args):
    fn = globals().get(name)
    if fn is None or not name.startswith("pase_spc_"):
        return emul_ops.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
