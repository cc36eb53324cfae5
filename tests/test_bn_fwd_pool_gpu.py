"""The summation order of the dense-skip pooling in the BatchNorm/PReLU forward pass.

Each pooled value is sum(a_t, t = w*pool_d .. (w+1)*pool_d - 1) * fp32(1 / pool_d), the sum taken
in fp32 in time order from 0 over exactly the values the kernel wrote to its operand (the
bf16-rounded ones in the bf16 format).  These tests rebuild that sum from the kernel's own
written rows and require the pooled output to match bit for bit, so a change to the kernel
cannot reorder the sum without failing here.  The other forward tests bound the window means
against float64 and check run-to-run repeatability, neither of which sees the order."""
import numpy as np
import pytest
import torch

from pase_b200 import _lib

pytestmark = pytest.mark.gpu

FMT_DT = {0: torch.float32, 1: torch.bfloat16}


def _rand(n, seed, scale=1.0, dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(n, generator=g)).to(dev)


def _params(C, seed):
    return _rand(C, seed), _rand(C, seed + 1), _rand(C, seed + 2, 0.3)


def _pool_ref(a, pool_d, pool_T):
    """a: [T, C] fp32 (CPU) operand rows of the unpadded frames -> [pool_T, C] fp32: each
    window summed in fp32 in time order from zero, times fp32(1/pool_d)."""
    inv_d = np.float32(1.0) / np.float32(pool_d)
    x = a.numpy().astype(np.float32)
    out = np.zeros((pool_T, x.shape[1]), np.float32)
    for w in range(pool_T):
        s = np.zeros(x.shape[1], np.float32)
        for t in range(w * pool_d, (w + 1) * pool_d):
            s = s + x[t]
        out[w] = s * inv_d
    return torch.from_numpy(out)


def _operand(dst, off, rows, rs, C):
    return torch.as_strided(dst, (rows, C), (rs, 1), off).float().cpu()


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("T,C,padL,padR,pool_d", [
    (203, 64, 4, 5, 1),
    (203, 64, 0, 0, 2),
    (205, 512, 5, 5, 4),
    (1001, 64, 3, 7, 8),
    (1003, 64, 5, 5, 16),
    (1607, 64, 125, 125, 160),     # block 0's window; T not a multiple of it, a long halo
    (1000, 64, 9, 1, 161),         # a window that is not a multiple of the chunk
    (999, 512, 0, 0, 161),
])
def test_pool_sum_order(T, C, padL, padR, pool_d, fmt):
    N = 2
    Tp = T + padL + padR
    pool_T = T // pool_d
    d_rs, p_rs = C + 8, C + 4
    d_ss, p_ss = (Tp + 1) * d_rs, (pool_T + 1) * p_rs
    y = _rand(N * T * C, 7 + pool_d)
    sc, sh, al = _params(C, 11)
    dst = torch.zeros(N * d_ss, dtype=FMT_DT[fmt], device="cuda")
    pool = torch.zeros(N * p_ss, device="cuda")
    _lib.call("pase_bn_prelu_pad_fwd", y, 0, T * C, N, T, C, sc, sh, al, dst, None, fmt,
              d_ss, d_rs, padL, padR, pool, p_ss, p_rs, pool_d, pool_T)
    torch.cuda.synchronize()
    for n in range(N):
        a = _operand(dst, n * d_ss + padL * d_rs, T, d_rs, C)
        got = _operand(pool, n * p_ss, pool_T, p_rs, C)
        ref = _pool_ref(a, pool_d, pool_T)
        assert torch.equal(got, ref), "sample %d: %d of %d pooled values differ" % (
            n, int((got != ref).sum()), got.numel())
        # rows past the pooled ones (and the pitch padding) stay untouched
        tail = pool[n * p_ss:(n + 1) * p_ss].view(pool_T + 1, p_rs)
        assert not bool(tail[:, C:].any()) and not bool(tail[pool_T].any())


@pytest.mark.parametrize("fmt", [0, 1])
def test_pool_sum_order_packed(fmt):
    """One pase_bn_prelu_pad_fwd_var launch over utterances of mixed lengths, each with its own
    pool_d and pool_T (some frames past the last window stay unpooled)."""
    C, padL, padR = 64, 5, 5
    Ts = [1607, 333, 170, 1003, 48, 2000]
    pds = [160, 8, 161, 16, 2, 1]
    pTs = [T // d for T, d in zip(Ts, pds)]
    pTs[-1] -= 3                                  # a tail of unpooled frames
    d_rs, p_rs = C, C + 4
    Tp = [T + padL + padR for T in Ts]
    y_off = np.concatenate([[0], np.cumsum(Ts)])[:-1] * C
    d_off = np.concatenate([[0], np.cumsum(np.asarray(Tp) + 1)])[:-1] * d_rs + d_rs
    p_off = np.concatenate([[0], np.cumsum(np.asarray(pTs) + 1)])[:-1] * p_rs
    tab = torch.tensor(np.stack([Ts, y_off, d_off, p_off, pds, pTs], 1).astype(np.int32)
                       .reshape(-1), device="cuda")
    y = _rand(sum(Ts) * C, 3)
    sc, sh, al = _params(C, 21)
    dst = torch.zeros(int(d_off[-1] + (Tp[-1] + 1) * d_rs), dtype=FMT_DT[fmt], device="cuda")
    pool = torch.zeros(int(p_off[-1] + (pTs[-1] + 1) * p_rs), device="cuda")
    _lib.call("pase_bn_prelu_pad_fwd_var", y, 0, tab, len(Ts), max(Ts), C, sc, sh, al, dst,
              None, fmt, d_rs, padL, padR, pool, p_rs, 1)
    torch.cuda.synchronize()
    for i, T in enumerate(Ts):
        a = _operand(dst, int(d_off[i]) + padL * d_rs, T, d_rs, C)
        got = _operand(pool, int(p_off[i]), pTs[i], p_rs, C)
        ref = _pool_ref(a, pds[i], pTs[i])
        assert torch.equal(got, ref), "utterance %d: %d of %d pooled values differ" % (
            i, int((got != ref).sum()), got.numel())
        assert not bool(_operand(pool, int(p_off[i]) + pTs[i] * p_rs, 1, p_rs, C).any())
