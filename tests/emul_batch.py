"""TEST-ONLY emulation of the batch-assembly entry points of include/pase_b200.h
(pase_b200/csrc/batch.cu) with torch's CPU fp32 operations, on CPU tensors.  ``call``
replaces ``pase_b200.ops.call`` (delegating the distortion entry points to emul_distort) so
that the host planner and orchestration of pase_b200/batch.py can be checked on a GPU-less
box.  Never imported by the product.
"""
import numpy as np
import torch

import emul_distort


def pase_chunk_gather(pcm, pcm_len, flt, flt_len, rows, B, nsrc, T, cchunk, out, plane):
    R = rows.reshape(B, nsrc, 6).tolist()
    flat = out.reshape(-1)
    for b in range(B):
        for s in range(nsrc):
            fmt, off, L, beg, scale, rbits = R[b][s]
            assert L >= 1 and (beg + T <= L or (beg == 0 and T - L < L))
            if fmt == 0:
                u = pcm[off:off + L].float() * (1.0 / 32768)
            else:
                u = flt[off:off + L]
            p = torch.arange(beg, beg + T)
            p = torch.where(p >= L, 2 * L - 2 - p, p)
            x = u[p]
            if scale:
                r = torch.from_numpy(np.array([rbits], np.int32).view(np.float32))
                x = x / torch.max(torch.abs(x)) * r
            flat[s * plane + b * T:s * plane + (b + 1) * T] = x
            if s == 0 and cchunk:
                flat[nsrc * plane + b * T:nsrc * plane + (b + 1) * T] = x


def pase_frames_gather(pool, pool_len, rows, B, F, n, out):
    for b, (off, frames, s) in enumerate(rows.reshape(B, 3).tolist()):
        assert s + n <= frames and off + F * frames <= pool_len
        X = pool[off:off + F * frames].view(F, frames)
        out[b].copy_(X[:, s:s + n])


def call(name, *args):
    fn = globals().get(name)
    if fn is not None:
        return fn(*args)
    return emul_distort.call(name, *args)
