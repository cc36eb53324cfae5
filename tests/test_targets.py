"""On-device LPS regression targets (SURVEY.md 8f N1): host logic on CPU with emulated kernels
against the oracle (torch.stft as the reference calls it + scipy's savgol for librosa.delta);
on the GPU the two new kernels against their spec and the whole transform against the oracle."""
import sys
import os

import numpy as np
import pytest
import torch

import emul
import pase_b200.ops as ops
from pase_b200.targets import LPS, savgol_taps

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import targets_oracle as TO                                   # noqa: E402


def _wave(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T) / 16000.0
    # noise + a few partials: bins span ~60 dB
    w = 0.1 * torch.randn(B, T, generator=g)
    for f, a in ((220.0, 0.5), (1870.0, 0.2), (5200.0, 0.05)):
        w += a * torch.sin(2 * np.pi * f * t)[None, :] * (1 + 0.3 * torch.rand(B, 1, generator=g))
    return w


def _check(got, wav, n_fft, hop, win, der, stats=None, tol_db=2e-3):
    """dB-scale comparison.  Both sides compute the spectrum in fp32-equivalent arithmetic:
    an amplitude error of ~5e-7 of the frame's largest component is a dB error of
    8.7 * 5e-7 * A_max / |X_k| at bin k (0.02 dB observed at a bin 104 dB below its frame's
    peak, from the oracle's fp32 FFT), on top of `tol_db`; delta rows are 9-tap combinations
    (sum |taps| < 0.5) of their bin's frames."""
    nb = n_fft // 2 + 1
    for b in range(wav.shape[0]):
        ref0 = TO.lps(wav[b], n_fft, hop, win, der)
        base = ref0[:nb]
        amp = 10.0 ** (base / 20.0)
        tol = tol_db + 8.7 * 5e-7 * amp.max(0, keepdim=True)[0] / amp
        tols = [tol] + [0.5 * tol.max(1, keepdim=True)[0].expand_as(tol)] * der
        tol = torch.cat(tols, 0)
        ref = ref0
        if stats is not None:
            ref = TO.znorm(ref0, stats[0], stats[1])
            tol = tol / stats[1].reshape(-1, 1)
        g = got[b].cpu()
        assert tuple(g.shape) == tuple(ref.shape)
        bad = (g - ref).abs() > tol
        assert not bool(bad.any()), (int(bad.sum()), float(((g - ref).abs() / tol).max()))


def test_savgol_taps_equal_scipy():
    from scipy.signal import savgol_filter
    x = np.random.RandomState(0).randn(4, 37)
    for width, order in ((9, 1), (9, 2), (5, 1), (7, 3)):
        taps = savgol_taps(width, order)
        ref = savgol_filter(x, width, deriv=order, polyorder=order, axis=-1, mode="interp")
        h = width // 2
        c = np.clip(np.arange(37), h, 36 - h)
        y = np.stack([(x[:, cc - h:cc + h + 1] * taps).sum(1) for cc in c], 1)
        assert np.abs(y - ref).max() < 1e-12


@pytest.mark.parametrize("T,win,der", [(3200, 400, 2), (4001, 512, 2), (1600, 400, 0)])
def test_lps_host_logic_against_oracle(monkeypatch, T, win, der):
    monkeypatch.setattr(ops, "call", emul.call)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    wav = _wave(2, T, 3)
    lps = LPS(n_fft=2048, hop=160, win=win, der_order=der, device="cpu")
    out = lps(wav.unsqueeze(1))
    assert tuple(out.shape) == (2, (1 + der) * 1025, T // 160)
    _check(out, wav, 2048, 160, win, der)
    # dict protocol + ZNorm folded in
    F = (1 + der) * 1025
    g = torch.Generator().manual_seed(9)
    stats = (torch.randn(F, generator=g) * 5 - 40, torch.rand(F, generator=g) * 10 + 2)
    lps2 = LPS(n_fft=2048, hop=160, win=win, der_order=der, name="lps_long", device="cpu",
               stats=stats)
    pkg = lps2({"chunk": wav[0]})
    assert pkg["dec_resolution"] == 160 and tuple(pkg["lps_long"].shape) == (F, T // 160)
    _check(pkg["lps_long"][None], wav[:1], 2048, 160, win, der, stats)


@pytest.mark.gpu
@pytest.mark.parametrize("N,T,win", [(3, 3200, 400), (2, 4001, 512)])
def test_lps_kernels_gpu(N, T, win):
    from pase_b200 import _lib
    hop, n_fft, lda = 160, 2048, -(-win // 64) * 64
    frames = T // hop
    x = _wave(N, T, 5).reshape(-1)
    start0 = (n_fft - win) // 2 - n_fft // 2
    hi, lo = (torch.zeros(N * frames * lda, dtype=torch.float16) for _ in range(2))
    emul.call("pase_frame_wave", x, N, T, hop, win, start0, frames, hi, lo, lda)
    dh, dl = hi.cuda().zero_(), lo.cuda().zero_()
    _lib.call("pase_frame_wave", x.cuda(), N, T, hop, win, start0, frames, dh, dl, lda)
    assert torch.equal(dh.cpu(), hi) and torch.equal(dl.cpu(), lo)
    nbins, ldc = 1025, 2052
    g = torch.Generator().manual_seed(6)
    C = torch.randn(N * frames * ldc, generator=g) * torch.logspace(-3, 1, N * frames * ldc)[
        torch.randperm(N * frames * ldc, generator=g)]
    fir = torch.from_numpy(np.stack([savgol_taps(9, d) for d in (1, 2)])).float().reshape(-1)
    F = 3 * nbins
    mean, std = torch.randn(F, generator=g), torch.rand(F, generator=g) + 0.5
    for st in (None, (mean, std)):
        ref = torch.zeros(N * F * frames)
        emul.call("pase_lps_post", C, ldc, N, frames, nbins, 2, 9, fir,
                  None if st is None else st[0], None if st is None else st[1], ref)
        out = torch.zeros(N * F * frames).cuda()
        _lib.call("pase_lps_post", C.cuda(), ldc, N, frames, nbins, 2, 9, fir.cuda(),
                  None if st is None else st[0].cuda(), None if st is None else st[1].cuda(), out)
        assert float((out.cpu() - ref).abs().max()) <= 2e-4 * (1.0 if st is None else 2.0)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,win", [(4, 32000, 400), (2, 32000, 512), (2, 48000, 400)])
def test_lps_gpu_against_oracle(B, T, win):
    wav = _wave(B, T, 11)
    lps = LPS(n_fft=2048, hop=160, win=win, der_order=2)
    out = lps(wav.cuda().unsqueeze(1))
    assert tuple(out.shape) == (B, 3075, T // 160)
    _check(out, wav, 2048, 160, win, 2)
