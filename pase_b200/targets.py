"""On-device regression targets (SURVEY.md 8f, N1): the log-power-spectrum label of the lps /
lps_long workers computed from the waveform chunks that are already in HBM, instead of on
DataLoader workers followed by a 79 MB host-to-device copy per label and step.

Mirrors ``pase.transforms.LPS`` (transforms.py:439-487: ``torch.stft(wav, n_fft, hop, win)`` with
the default rectangular window and centre reflect padding, ``10 log10(|X|^2 + 1e-19)``,
``librosa.feature.delta`` of orders 1..der_order stacked along the feature axis, first
``len // hop`` frames) and ``pase.transforms.ZNorm`` (transforms.py:183-202), batched:
(B, 1, T) chunks -> (B, (1 + der_order) * (n_fft/2 + 1), T // hop).

The STFT is one tensor-core GEMM (3xF16: fp32-equivalent products): only the `win` samples the
rectangular window keeps take part, so the n_fft-point transform of a frame is a
(win x 2*(n_fft/2+1)) real matrix product.  Kernels: csrc/targets.cu.
"""
import math

import numpy as np
import torch

from . import gemm, ops


def savgol_taps(width, order):
    """Correlation taps of ``scipy.signal.savgol_filter(x, width, polyorder=order, deriv=order,
    delta=1.0)`` -- what ``librosa.feature.delta(x, width=width, order=order)`` applies along
    time: the order-th derivative of the least-squares polynomial of degree `order` over the
    window (a constant over the window, which is also why mode='interp' reduces to clamping the
    window at the two edges).  float64 numpy, -> (width,) array with y[t] = sum_i taps[i] x[t-h+i]."""
    if width < 3 or width % 2 != 1 or not 1 <= order < width:
        raise ValueError("savgol_taps: odd width >= 3 and 1 <= order < width")
    h = width // 2
    pos = np.arange(-h, h + 1, dtype=np.float64)
    A = np.vander(pos, order + 1, increasing=True)           # columns 1, i, i^2, ...
    coef = np.linalg.pinv(A)                                 # (order+1, width): a_k = coef[k] . x
    return coef[order] * math.factorial(order)


class LPS(object):
    """``LPS(n_fft=2048, hop=160, win=400, der_order=2, name='lps')`` like the reference class;
    ``stats=(mean, std)`` (1-D tensors over the (1+der_order)*(n_fft/2+1) features, e.g. the
    entry of the reference's stats pickle) folds ZNorm into the same pass.

    ``lps(chunks)``: chunks (B, 1, T) / (B, T) / (T,) CUDA fp32 -> (B, F, T // hop) (a 1-D
    input returns (F, T // hop) like the reference).  ``lps(pkg)`` with a dict: reads
    ``pkg['chunk']`` and stores ``pkg[name]`` (+ ``pkg['dec_resolution'] = hop``)."""

    DELTA_WIDTH = 9                                          # librosa.feature.delta default

    def __init__(self, n_fft=2048, hop=160, win=400, der_order=2, name='lps', device='cuda',
                 stats=None):
        if win > n_fft or n_fft % 2:
            raise ValueError("LPS: need win <= n_fft and an even n_fft")
        self.n_fft, self.hop, self.win, self.der_order, self.name = n_fft, hop, win, der_order, name
        self.device = torch.device(device)
        self.nbins = n_fft // 2 + 1
        self.lda = -(-win // 64) * 64                        # operand row: multiple of 128 bytes
        self.ldc = -(-2 * self.nbins // 4) * 4
        self.stats = stats
        self._consts = None

    # ---- constants: DFT basis as an fp16-pair operand, delta filter taps ---------------
    def _build(self, dev):
        left = (self.n_fft - self.win) // 2                  # zero padding of the window
        m = np.arange(self.win, dtype=np.float64) + left
        k = np.arange(self.nbins, dtype=np.float64)
        ang = 2.0 * np.pi * np.outer(k, m) / self.n_fft
        basis = np.zeros((2 * self.nbins, self.lda), dtype=np.float64)
        basis[0::2, :self.win] = np.cos(ang)
        basis[1::2, :self.win] = -np.sin(ang)
        b32 = torch.from_numpy(basis).float().reshape(-1).to(dev)
        hi = torch.empty(b32.numel(), dtype=torch.float16, device=dev)
        lo = torch.empty_like(hi)
        ops.call("pase_split_f16", b32, hi, lo, b32.numel(), None, None)
        fir = None
        if self.der_order > 0:
            taps = np.stack([savgol_taps(self.DELTA_WIDTH, d) for d in range(1, self.der_order + 1)])
            fir = torch.from_numpy(taps).float().reshape(-1).to(dev)
        mean = std = None
        if self.stats is not None:
            mean = torch.as_tensor(self.stats[0], dtype=torch.float32).reshape(-1).to(dev)
            std = torch.as_tensor(self.stats[1], dtype=torch.float32).reshape(-1).to(dev)
            F = (1 + self.der_order) * self.nbins
            if mean.numel() != F or std.numel() != F:
                raise ValueError("LPS: stats must have %d entries" % F)
        self._consts = dict(dev=dev, hi=hi, lo=lo, fir=fir, mean=mean, std=std,
                            start0=left - self.n_fft // 2)

    def features(self, wav):
        """(B, T) CUDA fp32 -> (B, F, T // hop)."""
        if not wav.is_cuda:
            raise RuntimeError("pase_b200.targets.LPS runs on CUDA only (no CPU path); got %s"
                               % wav.device)
        wav = wav.contiguous().float()
        B, T = wav.shape
        frames = T // self.hop
        if frames < self.DELTA_WIDTH and self.der_order > 0:
            raise ValueError("LPS: %d frames are fewer than the delta window" % frames)
        dev = wav.device
        if self._consts is None or self._consts["dev"] != dev:
            self._build(dev)
        c = self._consts
        rows = B * frames
        a_hi = torch.empty(rows * self.lda, dtype=torch.float16, device=dev)
        a_lo = torch.empty_like(a_hi)
        ops.call("pase_frame_wave", wav.reshape(-1), B, T, self.hop, self.win, c["start0"], frames,
                 a_hi, a_lo, self.lda)
        spec = torch.empty(rows * self.ldc, dtype=torch.float32, device=dev)
        ops.call("pase_tc_gemm_nt", a_hi, a_lo, rows, self.lda, c["hi"], c["lo"], self.lda, spec,
                 self.ldc, rows, 2 * self.nbins, self.lda, 1.0, None, None, rows, rows, rows, 1,
                 None, None, 0, gemm.PRECISIONS["3xf16"].mode, 0)
        F = (1 + self.der_order) * self.nbins
        out = torch.empty(B, F, frames, dtype=torch.float32, device=dev)
        ops.call("pase_lps_post", spec, self.ldc, B, frames, self.nbins, self.der_order,
                 self.DELTA_WIDTH, c["fir"], c["mean"], c["std"], out.reshape(-1))
        return out

    def __call__(self, x):
        if isinstance(x, dict):
            wav = x["chunk"]
            x[self.name] = self(wav)
            x["dec_resolution"] = self.hop
            return x
        if x.dim() == 1:
            return self.features(x.reshape(1, -1))[0]
        if x.dim() == 3:
            if x.shape[1] != 1:
                raise ValueError("LPS: expected (B, 1, T) chunks, got %s" % (tuple(x.shape),))
            x = x[:, 0]
        return self.features(x)

    def __repr__(self):
        return "LPS(n_fft=%d, hop=%d, win=%d, device=%s)" % (self.n_fft, self.hop, self.win,
                                                             self.device)
