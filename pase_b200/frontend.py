"""Drop-in for ``pase.models.frontend`` (wf_builder / WaveFe, frontend.py:18-40,
116-279): same constructor kwargs, same ``state_dict`` keys and shapes, same
``forward(batch, device=None, mode=None)`` contract -- but forward and backward
run in the sm_90a kernels of ``pase_b200/csrc`` through ``pase_b200.encoder``.

The ``nn.Conv1d`` / ``nn.BatchNorm1d`` / ``nn.PReLU`` / ``nn.Linear`` objects
below are PARAMETER CONTAINERS only (they give the reference's key names and
default initialisation); their own ``forward`` is never called on this path.
"""
import json
import math
import os
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from .modules import Model, format_frontend_chunk, format_frontend_output
from . import encoder as _enc
from . import gemm as _gemm

# "3xtf32": wgmma tensor cores with error-compensated TF32 (fp32-equivalent, meets the
# fp32 parity bar); "fp32": FFMA kernels; "tf32": single-pass TF32 (L2-equivalent only).
# Shapes the tensor-core kernels cannot take (channel counts not multiples of 32) fall back
# to the FFMA kernels per GEMM -- still on the GPU, never to a CPU path.
# "auto": 3xF16 (fp32-equivalent products from fp16 operand pairs: half the tensor time and
# operand bytes of 3xTF32) when every channel count is a multiple of 64 (PASE.cfg, PASE+.cfg),
# else 3xTF32.  Both meet the fp32 parity bar (tests/test_encoder_gpu.py).
DEFAULT_PRECISION = "auto"

# Samples packed into one forward of WaveFe.extract (65.5 s of 16 kHz audio).  The packed plan
# this sizes holds 1.35 GB for PASE+ in 3xf16 and 0.75 GB in bf16 (EncoderPlan.nbytes() after a
# call, operand buffers included).
EXTRACT_MAX_SAMPLES = 1 << 20

_DEFAULTS = dict(
    num_inputs=1, sincnet=True,
    kwidths=[251, 10, 5, 5, 5, 5, 5, 5], strides=[1, 10, 2, 1, 2, 1, 2, 2],
    dilations=[1, 1, 1, 1, 1, 1, 1, 1],
    fmaps=[64, 64, 128, 128, 256, 256, 512, 512],
    norm_type="bnorm", pad_mode="reflect", sr=16000, emb_dim=256, rnn_dim=None,
    activation=None, rnn_pool=False, rnn_layers=1, rnn_dropout=0, rnn_type="qrnn",
    vq_K=None, vq_beta=0.25, vq_gamma=0.99, norm_out=False, tanh_out=False,
    resblocks=False, denseskips=False, densemerge="sum", name="WaveFe",
)


def wf_builder(cfg_path):
    """str path -> json -> WaveFe(**cfg); dict -> WaveFe(**cfg).  Named
    alternative encoders (asppRes / Resnet50 / tdnn, frontend.py:25-34) are other
    model families and are out of this package's scope."""
    if cfg_path is None:
        raise ValueError("cfg cannot be None!")
    if isinstance(cfg_path, str):
        with open(cfg_path, "r") as f:
            return wf_builder(json.load(f))
    if isinstance(cfg_path, dict):
        if "name" in cfg_path and cfg_path["name"] in ("asppRes", "Resnet50", "tdnn"):
            raise TypeError("Unrecognized frontend type for pase_b200: %s "
                            "(only the WaveFe encoder is implemented)" % cfg_path["name"])
        return WaveFe(**cfg_path)
    raise TypeError("Unexpected config for WaveFe")


class _SincParams(nn.Module):
    """low_hz_ / band_hz_ of SincConv_fast with its mel-scale initialisation
    (modules.py:853-866)."""

    def __init__(self, out_channels, kernel_size, sample_rate=16000,
                 min_low_hz=50, min_band_hz=50):
        super().__init__()
        if kernel_size % 2 == 0:
            kernel_size += 1
        self.out_channels, self.kernel_size = out_channels, kernel_size
        self.sample_rate, self.min_low_hz, self.min_band_hz = sample_rate, min_low_hz, min_band_hz
        mel = lambda hz: 2595 * np.log10(1 + hz / 700)
        edges = np.linspace(mel(30), mel(sample_rate / 2 - (min_low_hz + min_band_hz)),
                            out_channels + 1)
        hz = 700 * (10 ** (edges / 2595) - 1)
        self.low_hz_ = nn.Parameter(torch.Tensor(hz[:-1]).view(-1, 1))
        self.band_hz_ = nn.Parameter(torch.Tensor(np.diff(hz)).view(-1, 1))


class _FeBlock(nn.Module):
    def __init__(self, cin, cout, k, stride, sinc, sr):
        super().__init__()
        if sinc:
            if cin != 1:
                raise ValueError("SincConv only support one input channel "
                                 "(here, in_channels = {%i})" % cin)
            self.conv = _SincParams(cout, k, sample_rate=sr)
        else:
            self.conv = nn.Conv1d(cin, cout, k, stride)
        self.norm = nn.BatchNorm1d(cout)
        self.act = nn.PReLU(cout, init=0)


class _QRNNLayer(nn.Module):
    def __init__(self, in_size, hidden, window=2):
        super().__init__()
        self.linear = nn.Linear(window * in_size, 3 * hidden)


class _QRNN(nn.Module):
    def __init__(self, in_size, hidden):
        super().__init__()
        self.layers = nn.ModuleList([_QRNNLayer(in_size, hidden)])


class WaveFe(Model):
    """Convolutional waveform encoder (SincNet front + strided conv stack +
    optional dense skips, QRNN pooling and output BatchNorm)."""

    MAX_PLANS = 4

    def __init__(self, **kwargs):
        unknown = set(kwargs) - set(_DEFAULTS)
        if unknown:
            raise TypeError("WaveFe got unexpected arguments: %s" % sorted(unknown))
        cfg = dict(_DEFAULTS)
        cfg.update(kwargs)
        super().__init__(name=cfg["name"])
        self._check_supported(cfg)
        if cfg["rnn_pool"] and cfg["rnn_dim"] is None:
            cfg["rnn_dim"] = cfg["emb_dim"]
        self.cfg = cfg
        self.sincnet, self.kwidths = cfg["sincnet"], cfg["kwidths"]
        self.strides, self.fmaps = cfg["strides"], cfg["fmaps"]
        self.densemerge, self.rnn_pool = cfg["densemerge"], cfg["rnn_pool"]
        self.tanh_out, self.quantizer = False, None
        emb = cfg["emb_dim"]
        if cfg["denseskips"]:
            self.denseskips = nn.ModuleList()
        self.blocks = nn.ModuleList()
        cin = cfg["num_inputs"]
        n = len(cfg["kwidths"])
        for i, (k, s, f) in enumerate(zip(cfg["kwidths"], cfg["strides"], cfg["fmaps"])):
            self.blocks.append(_FeBlock(cin, f, k, s, cfg["sincnet"] and i == 0, cfg["sr"]))
            if cfg["denseskips"] and i + 1 < n:
                self.denseskips.append(nn.Conv1d(f, emb, 1, bias=False))
            cin = f
        if cfg["rnn_pool"]:
            self.rnn = _QRNN(cin, 2 * (cfg["rnn_dim"] // 2))
            self.W = nn.Conv1d(cfg["rnn_dim"], emb, 1)
        else:
            self.W = nn.Conv1d(cin, emb, 1)
        self.emb_dim = emb
        if cfg["norm_out"]:
            self.norm_out = nn.BatchNorm1d(emb, affine=False)
        self._plans = OrderedDict()
        self._packed_plans = OrderedDict()
        # GEMM numerics (gemm.PRECISIONS): "fp32" (FFMA), "3xtf32" / "3xf16" (wgmma,
        # fp32-equivalent), "tf32" (wgmma), "bf16" (wgmma, bf16 operands and activations)
        self.precision = os.environ.get("PASE_B200_PRECISION", DEFAULT_PRECISION)
        self._sinc_n = self._sinc_win = None
        self.last_output_ntc = None

    @staticmethod
    def _check_supported(cfg):
        def need(cond, what):
            if not cond:
                raise NotImplementedError(
                    "pase_b200.WaveFe: %s is not implemented natively (PASE.cfg / PASE+.cfg "
                    "feature set only); refusing to fall back." % what)
        need(cfg["sincnet"], "sincnet=False")
        need(cfg["num_inputs"] == 1, "num_inputs != 1")
        need(cfg["norm_type"] == "bnorm", "norm_type=%r" % cfg["norm_type"])
        need(cfg["pad_mode"] == "reflect", "pad_mode=%r" % cfg["pad_mode"])
        need(cfg["activation"] in (None, "prelu"), "activation=%r" % cfg["activation"])
        need(all(d == 1 for d in cfg["dilations"][:len(cfg["kwidths"])]), "dilation > 1")
        need(not cfg["resblocks"], "resblocks")
        need(cfg["vq_K"] in (None, 0), "vector quantizer")
        need(not cfg["tanh_out"], "tanh_out")
        need(cfg["densemerge"] == "sum", "densemerge=%r" % cfg["densemerge"])
        need(cfg["strides"][0] == 1, "strided sinc layer")
        if cfg["rnn_pool"]:
            need(cfg["rnn_type"].lower() == "qrnn", "rnn_type=%r" % cfg["rnn_type"])
            need(cfg["rnn_layers"] == 1, "rnn_layers != 1")
            need(cfg["rnn_dropout"] == 0, "rnn_dropout")
        assert len(cfg["kwidths"]) == len(cfg["strides"]) == len(cfg["fmaps"])
        need(all(f % 4 == 0 for f in cfg["fmaps"]) and cfg["emb_dim"] % 4 == 0,
             "channel counts that are not multiples of 4")

    # -- engine plumbing ---------------------------------------------------
    def resolved_precision(self):
        if self.precision != "auto":
            return self.precision
        wide = all(f % 64 == 0 for f in self.cfg["fmaps"])
        return "3xf16" if wide else "3xtf32"

    def _plan(self, N, T, device):
        prec = self.resolved_precision()
        key = (N, T, str(device), prec)
        plan = self._plans.get(key)
        if plan is None:
            plan = _enc.EncoderPlan(self.cfg, N, T, device, prec)
            self._plans[key] = plan
            while len(self._plans) > self.MAX_PLANS:
                self._plans.popitem(last=False)
        else:
            self._plans.move_to_end(key)
        return plan

    def _packed_plan(self, capacity, device):
        prec = self.resolved_precision()
        key = (capacity, str(device), prec)
        plan = self._packed_plans.get(key)
        if plan is None:
            plan = _enc.PackedPlan(self.cfg, capacity, device, prec)
            self._packed_plans[key] = plan
            while len(self._packed_plans) > self.MAX_PLANS:
                self._packed_plans.popitem(last=False)
        else:
            self._packed_plans.move_to_end(key)
        return plan

    def _sinc_consts(self, device):
        if self._sinc_n is None or self._sinc_n.device != device:
            k = self.blocks[0].conv.kernel_size
            self._sinc_n, self._sinc_win = _enc.sinc_constants(k, self.cfg["sr"], device)

    def encode(self, x):
        """(N,1,T) CUDA fp32 tensor -> (out (N,emb,T'), out_ntc (N*T',emb))."""
        if x.dim() != 3 or x.shape[1] != 1:
            raise ValueError("WaveFe expects (N,1,T) waveforms, got %s" % (tuple(x.shape),))
        if not x.is_cuda:
            raise RuntimeError("pase_b200.WaveFe runs on CUDA (sm_90a) only; got a %s tensor. "
                               "There is no CPU path." % x.device)
        x = x.contiguous().float()
        self._sinc_consts(x.device)
        plan = self._plan(x.shape[0], x.shape[2], x.device)
        named = [(n, p) for n, p in self.named_parameters()]
        names = tuple(n for n, _ in named)
        tensors = [p for _, p in named]
        if tensors and tensors[0].device != x.device:
            raise RuntimeError("WaveFe parameters live on %s but the input is on %s"
                               % (tensors[0].device, x.device))
        if torch.is_grad_enabled() and any(p.requires_grad for p in tensors):
            plan.ensure_backward()
            return _enc._EncoderFn.apply(x, self, plan, self.training, names, *tensors)
        with torch.no_grad():
            return _enc.encoder_forward(plan, self, x, dict(named), self.training, False)

    def extract(self, wavs, mode=None, max_samples=None):
        """Features of many utterances of any lengths, packed into as few forwards as fit
        `max_samples` samples each (default EXTRACT_MAX_SAMPLES; greedy, in order; a longer
        utterance gets a forward of its own).  wavs: list of fp32 (T,), (1,T) or (1,1,T)
        tensors, on the CPU or the GPU.  Returns, in input order, (1, emb', T'_i) CUDA tensors
        equal to ``self(wavs[i].view(1,1,-1), mode=mode)`` (mode as select_output); they are
        views of one buffer per forward.  Eval mode only: train-mode BatchNorm would couple
        the utterances."""
        if self.training:
            raise RuntimeError("WaveFe.extract runs the encoder in eval mode; call .eval() first "
                               "(train-mode BatchNorm statistics would mix the utterances)")
        device = self.W.weight.device
        if device.type != "cuda":
            raise RuntimeError("pase_b200.WaveFe runs on CUDA (sm_90a) only; the module lives "
                               "on %s. There is no CPU path." % device)
        return self._extract(wavs, mode, max_samples, device)

    def _extract(self, wavs, mode, max_samples, device):
        if mode not in _enc.OUT_MODES:
            raise ValueError("mode must be one of %s, got %r" % (list(_enc.OUT_MODES), mode))
        cap = EXTRACT_MAX_SAMPLES if max_samples is None else int(max_samples)
        if cap < 1:
            raise ValueError("max_samples must be positive, got %r" % (max_samples,))
        flat = []
        for i, w in enumerate(wavs):
            if not isinstance(w, torch.Tensor) or w.dtype != torch.float32:
                raise TypeError("utterance %d: expected an fp32 tensor, got %s"
                                % (i, getattr(w, "dtype", type(w))))
            if w.dim() == 0 or w.dim() > 3 or any(d != 1 for d in w.shape[:-1]):
                raise ValueError("utterance %d: expected (T,), (1,T) or (1,1,T), got %s"
                                 % (i, tuple(w.shape)))
            flat.append(w.reshape(-1))
        if not flat:
            return []
        lengths = [w.numel() for w in flat]
        fold = _gemm.PRECISIONS[self.resolved_precision()].sinc_fold
        geoms = _enc.utterance_geometry(self.cfg, lengths, fold)
        self._sinc_consts(device)
        params = dict(self.named_parameters())
        feats = []
        with torch.no_grad():
            for a, b in _enc.split_packs(lengths, cap):
                total = sum(lengths[a:b])
                plan = self._packed_plan(max(cap, total), device)
                x = plan.wave[:total]
                if all(not w.is_cuda for w in flat[a:b]):
                    x.copy_(torch.cat(flat[a:b]))
                else:
                    torch.cat([w.to(device) for w in flat[a:b]], out=x)
                feats += _enc.encoder_forward_packed(plan, self, x, lengths[a:b], geoms[a:b],
                                                     params, mode)
        return feats

    def forward(self, batch, device=None, mode=None):
        if device is None:
            # Model.parameters() only yields trainable parameters: a frozen encoder (a fixed
            # feature extractor downstream) must still resolve its device
            device = self.W.weight.device
        x, data_fmt = format_frontend_chunk(batch, device)
        if not x.is_cuda:
            x = x.to(device)
        out, out_ntc = self.encode(x)
        self.last_output_ntc = out_ntc
        return format_frontend_output(out, data_fmt, mode)

    def frame_counts(self, T):
        return _enc.frame_counts(self.cfg, T)
