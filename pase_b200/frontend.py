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
from . import ops as _ops

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

# Samples whose frames one segment of WaveFe.extract_long computes (65.5 s of 16 kHz audio).
EXTRACT_LONG_WINDOW = 1 << 20

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
        self._stagers, self._carries = {}, {}
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

    def _eval_device(self, what):
        if self.training:
            raise RuntimeError("WaveFe.%s runs the encoder in eval mode; call .eval() first"
                               % what)
        device = self.W.weight.device
        if device.type != "cuda":
            raise RuntimeError("pase_b200.WaveFe runs on CUDA (sm_90a) only; the module lives "
                               "on %s. There is no CPU path." % device)
        return device

    def extract_long(self, wav, mode=None, window=None):
        """Features of one recording of any length in memory bounded by the window: (1, emb',
        T') CUDA tensor equal to ``self(wav.view(1,1,-1), mode=mode)``.  The recording is cut
        into segments whose crops hold `window` samples' frames (default EXTRACT_LONG_WINDOW,
        at least encoder.min_window), each with halos covering the receptive field, and the
        QRNN state is carried from one to the next (DESIGN.md section 15).  A recording of at
        most `window` samples runs as one forward of `extract`.  wav: fp32 (T,), (1,T) or
        (1,1,T) on the CPU (staged segment by segment through pinned memory) or the GPU.
        Eval mode only."""
        return self._extract_long(wav, mode, window, self._eval_device("extract_long"))

    def _extract_long(self, wav, mode, window, device):
        if mode not in _enc.OUT_MODES:
            raise ValueError("mode must be one of %s, got %r" % (list(_enc.OUT_MODES), mode))
        x = _recording(wav)
        win = EXTRACT_LONG_WINDOW if window is None else int(window)
        cfg, L = self.cfg, x.numel()
        if win < _enc.min_window(cfg):
            raise ValueError("window must be at least %d samples, got %d"
                             % (_enc.min_window(cfg), win))
        if L <= win:
            return self._extract([x], mode, win, device)[0]
        segs = _enc.plan_windows(cfg, L, win)            # every check before the first launch
        T = _enc.frame_counts(cfg, L)[-1]
        emb = self.emb_dim
        E = emb * (2 if mode in ("avg_concat", "avg_norm_concat") else 1)
        plan = self._packed_plan(_enc.window_capacity(cfg, win), device)
        fold = plan.precision.sinc_fold
        stage = None
        if device.type == "cuda" and not x.is_cuda:
            stage = self._stager(plan.capacity)
        elif x.device != device:
            x = x.to(device)
        self._sinc_consts(device)
        params = dict(self.named_parameters())
        out = torch.empty(E, T, dtype=torch.float32, device=device)
        carry = self._carry(plan, device)
        col = 0
        with torch.no_grad():
            for seg in segs:
                s, n = seg["seg_start"], seg["seg_len"]
                xs = x[s:s + n] if stage is None else stage.put(x[s:s + n], plan.wave)
                _enc.encoder_forward_window(plan, self, xs, seg,
                                            _enc.build_geometry(cfg, n, fold), params, carry,
                                            out, T, col)
                col += seg["crop_n"]
            if mode is not None:
                _ops.call("pase_out_select", out, T, emb, _enc.OUT_MODES[mode])
        return out.view(1, E, T)

    def stream(self, mode=None, window=None):
        """A FeatureStream over this encoder: push() samples as they arrive, get back the
        frames that are already final.  Eval mode only, mode None only (the avg modes need the
        whole recording)."""
        device = self._eval_device("stream")
        if mode is not None:
            raise ValueError("a FeatureStream returns mode None features only; select_output "
                             "modes need the whole recording (use extract_long)")
        return FeatureStream(self, device, window)

    def _stager(self, n):
        st = self._stagers.get(n)
        if st is None:
            st = self._stagers[n] = _PinnedStager(n)
        return st

    def _carry(self, plan, device):
        """Zeroed QRNN state of a windowed forward (one buffer per device, reused)."""
        if not plan.rnn:
            return None
        c = self._carries.get(str(device))
        if c is None or c.numel() != plan.H:
            c = self._carries[str(device)] = torch.zeros(plan.H, dtype=torch.float32,
                                                         device=device)
        return c.zero_()

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


def _recording(w):
    """One fp32 recording as (T,), (1,T) or (1,1,T) -> its flat contiguous (T,) view."""
    if not isinstance(w, torch.Tensor) or w.dtype != torch.float32:
        raise TypeError("expected an fp32 tensor, got %s" % getattr(w, "dtype", type(w)))
    if w.dim() == 0 or w.dim() > 3 or any(d != 1 for d in w.shape[:-1]):
        raise ValueError("expected a (T,), (1,T) or (1,1,T) recording, got %s"
                         % (tuple(w.shape),))
    return w.reshape(-1).contiguous()


class _PinnedStager(object):
    """Two pinned host buffers of n floats: a CPU segment is copied into one while the device
    may still be reading the other, then sent to the device asynchronously."""

    def __init__(self, n):
        self.bufs = [torch.empty(n, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.events = [None, None]
        self.i = 0

    def put(self, src, dst):
        i, self.i = self.i, self.i ^ 1
        if self.events[i] is not None:
            self.events[i].synchronize()          # its last copy to the device has finished
        n = src.numel()
        self.bufs[i][:n].copy_(src)
        d = dst[:n]
        d.copy_(self.bufs[i][:n], non_blocking=True)
        self.events[i] = torch.cuda.Event()
        self.events[i].record()
        return d


class FeatureStream(object):
    """Online feature extraction of one recording (WaveFe.stream()).  push(samples) returns the
    (1, emb, n) frames that became final (n may be 0): frame j is final once sample
    hop*j + B has arrived (B: encoder.receptive_field, 1335 samples for PASE+) and at least
    encoder.tail_length samples have.  finish() returns the rest, the end of the recording
    reflect-padded as a whole-recording forward pads it.  The frames concatenate to
    ``WaveFe.extract_long`` of the whole recording (bit-equal when it has more than 512
    frames, where both run the sequential QRNN scan).  Between calls the stream holds only the
    samples its next segment reads again (halo and tail), the QRNN state and frame counters."""

    def __init__(self, model, device, window=None):
        cfg = model.cfg
        win = _enc.min_window(cfg) if window is None else int(window)
        if win < _enc.min_window(cfg):
            raise ValueError("window must be at least %d samples, got %d"
                             % (_enc.min_window(cfg), win))
        self.model, self.device, self.cfg = model, device, cfg
        self.chunk = win // _enc.hop_size(cfg) * _enc.hop_size(cfg)
        self.min_len = _enc.min_length(cfg)
        self.plan = model._packed_plan(_enc.window_capacity(cfg, win), device)
        self.carry = (torch.zeros(self.plan.H, dtype=torch.float32, device=device)
                      if self.plan.rnn else None)
        self.buf = None            # samples buf0 .. n-1 (the ones a later segment reads)
        self.buf0 = 0
        self.n = 0                 # samples received
        self.done = 0              # frames returned
        self.finished = False

    def push(self, samples):
        if self.finished:
            raise RuntimeError("FeatureStream.push after finish()")
        x = _recording(samples)
        outs = []
        for a in range(0, x.numel(), self.chunk):
            piece = x[a:a + self.chunk]
            self.buf = piece.clone() if self.buf is None else torch.cat([self.buf,
                                                                         piece.to(self.buf)])
            self.n += piece.numel()
            f1 = _enc.final_frames(self.cfg, self.n)
            if f1 > self.done:
                outs.append(self._run(f1, False))
        if not outs:
            return torch.empty(1, self.model.emb_dim, 0, dtype=torch.float32, device=self.device)
        return outs[0] if len(outs) == 1 else torch.cat(outs, 2)

    def finish(self):
        if self.finished:
            raise RuntimeError("FeatureStream.finish called twice")
        if self.n < self.min_len:
            raise ValueError("a recording of %d samples is shorter than the encoder's minimum "
                             "of %d" % (self.n, self.min_len))
        if self.done > 0:
            _enc.check_windowable(self.cfg, self.n)
        self.finished = True
        T = _enc.frame_counts(self.cfg, self.n)[-1]
        if T > self.done:
            return self._run(T, True)
        return torch.empty(1, self.model.emb_dim, 0, dtype=torch.float32, device=self.device)

    def _run(self, f1, at_end):
        cfg, plan, m = self.cfg, self.plan, self.model
        seg = _enc.make_segment(cfg, self.done, f1,
                                self.n if at_end else _enc.stream_end(cfg, self.n))
        _enc.check_segment(cfg, seg, at_end)
        s, n = seg["seg_start"], seg["seg_len"]
        assert s >= self.buf0 and n <= plan.capacity
        x = plan.wave[:n]
        x.copy_(self.buf[s - self.buf0:s - self.buf0 + n])
        out = torch.empty(m.emb_dim, f1 - self.done, dtype=torch.float32, device=self.device)
        m._sinc_consts(self.device)
        with torch.no_grad():
            _enc.encoder_forward_window(
                plan, m, x, seg, _enc.build_geometry(cfg, n, plan.precision.sinc_fold),
                dict(m.named_parameters()), self.carry, out, f1 - self.done, 0)
        self.done = f1
        # keep what the next segment can read: from its left halo or its tail extension
        hop = _enc.hop_size(cfg)
        keep = min(max(0, self.done - _enc.window_halos(cfg)[0]) * hop,
                   max(0, (_enc.stream_end(cfg, self.n) - _enc.tail_length(cfg)) // hop * hop))
        if keep > self.buf0:
            self.buf = self.buf[keep - self.buf0:].clone()
            self.buf0 = keep
        return out.view(1, m.emb_dim, -1)
