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

# Samples packed into one forward of a StreamPool round: every segment holds at least
# encoder.tail_length samples (24310 for PASE+), so a pack serves about 43 streams (DESIGN.md
# section 16).  The plan it sizes is that of WaveFe.extract.
STREAM_POOL_MAX_SAMPLES = EXTRACT_MAX_SAMPLES

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
        self._grad_plans = OrderedDict()       # encode_packed: apart from extract's plans
        self._long_pool = None          # (key, StreamPool) of extract_long
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

    def _cached_plan(self, cache, key, build):
        """cache[key], built by build() on a miss; the cache keeps the MAX_PLANS most recently
        used plans."""
        plan = cache.get(key)
        if plan is None:
            plan = cache[key] = build()
            while len(cache) > self.MAX_PLANS:
                cache.popitem(last=False)
        else:
            cache.move_to_end(key)
        return plan

    def _plan(self, N, T, device):
        prec = self.resolved_precision()
        return self._cached_plan(self._plans, (N, T, str(device), prec),
                                 lambda: _enc.EncoderPlan(self.cfg, N, T, device, prec))

    def _packed_plan(self, capacity, device):
        prec = self.resolved_precision()
        return self._cached_plan(self._packed_plans, (capacity, str(device), prec),
                                 lambda: _enc.PackedPlan(self.cfg, capacity, device, prec))

    def _grad_plan(self, capacity, device):
        prec = self.resolved_precision()
        return self._cached_plan(self._grad_plans, (capacity, prec, str(device)),
                                 lambda: _enc.PackedGradPlan(self.cfg, capacity, device, prec))

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
        return self._encode(x.contiguous().float())

    def _encode(self, x):
        """encode past its checks on the input: differentiated (the _EncoderFn node) when grad
        mode is on and the waveform or a parameter needs a gradient, else the forward alone."""
        self._sinc_consts(x.device)
        plan = self._plan(x.shape[0], x.shape[2], x.device)
        named = [(n, p) for n, p in self.named_parameters()]
        names = tuple(n for n, _ in named)
        tensors = [p for _, p in named]
        if tensors and tensors[0].device != x.device:
            raise RuntimeError("WaveFe parameters live on %s but the input is on %s"
                               % (tensors[0].device, x.device))
        if torch.is_grad_enabled() and (x.requires_grad or
                                        any(p.requires_grad for p in tensors)):
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
        return self._extract(wavs, mode, max_samples, self._eval_device("extract"))

    def _extract(self, wavs, mode, max_samples, device):
        if mode not in _enc.OUT_MODES:
            raise ValueError("mode must be one of %s, got %r" % (list(_enc.OUT_MODES), mode))
        cap = self._packed_cap(max_samples)
        flat = self._packed_inputs(wavs)
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

    def encode_packed(self, wavs, max_samples=None):
        """Differentiable packed encoding of utterances of any lengths (DESIGN.md section 18):
        wavs as in extract; returns, in input order, the (1, emb, T'_i) CUDA tensors of
        ``extract(wavs, mode=None)`` (the same launches and bits).  With grad mode on and a
        waveform or a parameter requiring a gradient, one autograd node backpropagates to every
        waveform (through the caller's own .to() / .view()) and to the parameters (summed over
        the utterances; autograd or grad_sink).  One pack per call: the total must fit
        `max_samples` (default EXTRACT_MAX_SAMPLES).  Eval mode only."""
        device = self._eval_device("encode_packed")
        cap = self._packed_cap(max_samples)
        flat = self._packed_inputs(wavs)
        if not flat:
            return []
        return self._encode_packed(flat, cap, device)

    def encode_packed_train(self, wavs, max_samples=None):
        """Train-mode packed encoding (DESIGN.md section 19): wavs and the returned (1, emb,
        T'_i) CUDA views of one buffer as in encode_packed.  Every BatchNorm (each block's and
        norm_out) normalises with the mean and biased variance over the valid frames of all
        utterances, i.e. as nn.BatchNorm1d on their time-concatenation (1, C, sum T_i), and
        updates its running statistics and num_batches_tracked once per call (also under
        no_grad).  No padding enters the statistics, so with equal lengths this is the train
        forward of the stacked (N, 1, T) batch.  With grad mode on and a waveform or a parameter
        requiring a gradient, one autograd node backpropagates through the batch statistics to
        every waveform and to the parameters (autograd or grad_sink, all or nothing as in
        encode).  One pack per call: the total must fit `max_samples` (default
        EXTRACT_MAX_SAMPLES).  Train mode only; everything is checked before any launch."""
        if not self.training:
            raise RuntimeError("WaveFe.encode_packed_train runs the encoder in train mode; in "
                               "eval mode use encode_packed")
        device = self._device()
        flat = self._packed_inputs(wavs)
        if not flat:
            return []
        return self._encode_packed(flat, self._packed_cap(max_samples), device, True)

    def _packed_cap(self, max_samples):
        cap = EXTRACT_MAX_SAMPLES if max_samples is None else int(max_samples)
        if cap < 1:
            raise ValueError("max_samples must be positive, got %r" % (max_samples,))
        return cap

    @staticmethod
    def _packed_inputs(wavs):
        flat = []
        for i, w in enumerate(wavs):
            try:
                flat.append(_recording(w))
            except (TypeError, ValueError) as e:
                raise type(e)("utterance %d: %s" % (i, e)) from None
        return flat

    def _encode_packed(self, flat, cap, device, training=False):
        lengths = [w.numel() for w in flat]
        what = "encode_packed_train" if training else "encode_packed"
        if sum(lengths) > cap:
            raise ValueError("%s: %d samples exceed max_samples=%d; one call is one "
                             "pack, so split the list into calls that fit"
                             % (what, sum(lengths), cap))
        if len(lengths) > _enc.MAX_UTTS:
            raise ValueError("%s: %d utterances exceed the %d of one pack; split the list into "
                             "calls that fit" % (what, len(lengths), _enc.MAX_UTTS))
        fold = _gemm.PRECISIONS[self.resolved_precision()].sinc_fold
        geoms = _enc.utterance_geometry(self.cfg, lengths, fold)
        self._sinc_consts(device)
        plan = self._grad_plan(cap, device)
        named = list(self.named_parameters())
        names = tuple(n for n, _ in named)
        tensors = [p for _, p in named]
        xs = [w.to(device) for w in flat]
        if torch.is_grad_enabled() and (any(w.requires_grad for w in xs) or
                                        any(p.requires_grad for p in tensors)):
            return list(_enc._PackedEncoderFn.apply(self, plan, lengths, geoms, names, training,
                                                    len(xs), *xs, *tensors))
        with torch.no_grad():
            x = plan.wave[:sum(lengths)]
            torch.cat(xs, out=x)
            return _enc.encoder_forward_packed(plan, self, x, lengths, geoms, dict(named),
                                               training=training)

    def _eval_device(self, what):
        if self.training:
            raise RuntimeError("WaveFe.%s runs the encoder in eval mode; call .eval() first"
                               % what)
        return self._device()

    def _device(self):
        """The module's device, which must be a CUDA one."""
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
        QRNN state is carried from one to the next (DESIGN.md section 15): the recording runs
        as one push of a one-stream StreamPool, finished in the same call.  A recording of at
        most `window` samples runs as one forward of `extract`.  wav: fp32 (T,), (1,T) or
        (1,1,T) on the CPU (staged piece by piece through pinned memory) or the GPU.
        Eval mode only."""
        return self._extract_long(wav, mode, window, self._eval_device("extract_long"))

    def _extract_long(self, wav, mode, window, device):
        if mode not in _enc.OUT_MODES:
            raise ValueError("mode must be one of %s, got %r" % (list(_enc.OUT_MODES), mode))
        x = _recording(wav)
        cfg, L = self.cfg, x.numel()
        win = _check_window(cfg, EXTRACT_LONG_WINDOW if window is None else window)
        if L <= win:
            return self._extract([x], mode, win, device)[0]
        if x.is_cuda and x.device != device:
            x = x.to(device)
        T, emb = _enc.frame_counts(cfg, L)[-1], self.emb_dim
        E = emb * (2 if mode in ("avg_concat", "avg_norm_concat") else 1)
        pool = self._long_stream_pool(win, device)
        out = torch.empty(E, T, dtype=torch.float32, device=device)
        sid = pool.open()
        try:                        # the whole recording as one push: plan_windows' segments
            pool._push({sid: x}, [sid], out)
        finally:
            pool._release(sid)      # a no-op once the push has finished the stream
        if mode is not None:
            _ops.call("pase_out_select", out, T, emb, _enc.OUT_MODES[mode])
        return out.view(1, E, T)

    def _long_stream_pool(self, win, device):
        """The cached one-stream pool (its ring and staging) of extract_long and encode_long,
        one per (window, device, precision)."""
        key = (win, str(device), self.resolved_precision())
        if self._long_pool is None or self._long_pool[0] != key:
            self._long_pool = None
            self._long_pool = (key, StreamPool(self, device, 1, win,
                                               _enc.window_capacity(self.cfg, win)))
        return self._long_pool[1]

    def encode_long(self, wav, window=None):
        """Differentiable encoding of one recording of any length in bounded memory (DESIGN.md
        section 20).  wav: fp32 (T,), (1,T) or (1,1,T) on the module's CUDA device.  Returns the
        (1, emb, T') features of ``extract_long(wav, mode=None, window=window)``: the same
        segments and bits.  With grad mode on and the waveform or a parameter requiring a
        gradient, one autograd node backpropagates to the waveform and to the parameters
        (summed over the recording; autograd or grad_sink, all or nothing as in encode; a frozen
        encoder runs the data-gradient sweep only).  Its backward recomputes one window at a
        time on the PackedGradPlan of encoder.window_capacity(window) samples, which it may
        share with encode_packed: running it bumps that plan's generation, so a pending
        encode_packed backward on the same plan raises.  Memory is bounded by that plan, the
        forward's plan and O(T) tensors.  A recording of at most `window` samples is
        ``encode_packed([wav], max_samples=window)[0]``.  Eval mode only; select_output modes are
        torch ops on the result.  Everything is checked before any launch."""
        return self._encode_long(wav, window, self._eval_device("encode_long"))

    def _encode_long(self, wav, window, device):
        x = _recording(wav)
        if x.device != device:
            raise RuntimeError("WaveFe.encode_long: the recording lives on %s, the module on "
                               "%s; move it to the module's device (its gradient is returned "
                               "there)" % (x.device, device))
        cfg, L = self.cfg, x.numel()
        win = _check_window(cfg, EXTRACT_LONG_WINDOW if window is None else window)
        if L < _enc.min_length(cfg):
            raise ValueError("a recording of %d samples is shorter than the encoder's minimum "
                             "of %d" % (L, _enc.min_length(cfg)))
        if L <= win:
            return self._encode_packed([x], win, device)[0]
        _enc.check_windowable(cfg, L)
        segs = _enc.plan_windows(cfg, L, win)
        named = list(self.named_parameters())
        names = tuple(n for n, _ in named)
        tensors = [p for _, p in named]
        pool = self._long_stream_pool(win, device)
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in tensors)):
            return _enc._LongEncoderFn.apply(self, pool, win, segs, names, x, *tensors)
        T = _enc.frame_counts(cfg, L)[-1]
        out = torch.empty(self.emb_dim, T, dtype=torch.float32, device=device)
        sid = pool.open()
        try:
            with torch.no_grad():
                pool._push({sid: x}, [sid], out)
        finally:
            pool._release(sid)
        return out.view(1, self.emb_dim, T)

    def stream(self, mode=None, window=None):
        """A FeatureStream over this encoder: push() samples as they arrive, get back the
        frames that are already final.  Eval mode only, mode None only (the avg modes need the
        whole recording)."""
        device = self._eval_device("stream")
        if mode is not None:
            raise ValueError("a FeatureStream returns mode None features only; select_output "
                             "modes need the whole recording (use extract_long)")
        return FeatureStream(self, device, window)

    def streams(self, max_streams, window=None, max_samples=None, mode=None):
        """A StreamPool of up to `max_streams` live recordings at once: each push() runs every
        stream's next segment in one packed forward per round (at most `max_samples` samples
        per forward, default STREAM_POOL_MAX_SAMPLES), and each stream's frames are those of a
        FeatureStream fed the same blocks.  Eval mode only, mode None only."""
        device = self._eval_device("streams")
        if mode is not None:
            raise ValueError("a FeatureStream returns mode None features only; select_output "
                             "modes need the whole recording (use extract_long)")
        return StreamPool(self, device, max_streams, window, max_samples)

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


def _check_window(cfg, window):
    """A window of `window` samples (int), refused below encoder.min_window."""
    win = int(window)
    if win < _enc.min_window(cfg):
        raise ValueError("window must be at least %d samples, got %d"
                         % (_enc.min_window(cfg), win))
    return win


class FeatureStream(object):
    """Online feature extraction of one recording (WaveFe.stream()).  push(samples) returns the
    (1, emb, n) frames that became final (n may be 0): frame j is final once sample
    hop*j + B has arrived (B: encoder.receptive_field, 1335 samples for PASE+) and at least
    encoder.tail_length samples have.  finish() returns the rest, the end of the recording
    reflect-padded as a whole-recording forward pads it.  The frames concatenate to
    ``WaveFe.extract_long`` of the whole recording (bit-equal when it has more than 512
    frames, where both run the sequential QRNN scan).  A stream is one open id of a private
    one-stream StreamPool whose plan holds the longest segment of its window
    (encoder.window_capacity): between calls the device holds the samples a later segment reads
    again and the QRNN state, the host four counters."""

    def __init__(self, model, device, window=None):
        win = _enc.min_window(model.cfg) if window is None else int(window)
        self._pool = StreamPool(model, device, 1, win, _enc.window_capacity(model.cfg, win))
        self._id = self._pool.open()
        self.finished = False

    def push(self, samples):
        if self.finished:
            raise RuntimeError("FeatureStream.push after finish()")
        return self._pool.push({self._id: samples})[self._id]

    def finish(self):
        if self.finished:
            raise RuntimeError("FeatureStream.finish called twice")
        out = self._pool.push({}, finish=[self._id])[self._id]
        self.finished = True
        return out


class _PoolStream(object):
    """Host counters of one pooled stream: its ring slot, samples received, frames returned and
    the first sample it still holds."""
    __slots__ = ("slot", "n", "done", "keep")

    def __init__(self, slot):
        self.slot, self.n, self.done, self.keep = slot, 0, 0, 0


class StreamPool(object):
    """Online feature extraction of many live recordings at once (WaveFe.streams()).

    open() returns a stream id; push({id: samples, ...}, finish=(ids...)) returns {id: (1, emb,
    n) frames} for every id named, n >= 0.  Every stream is planned by the host planner
    encoder.stream_step, one piece of at most stream_chunk samples at a time; a stream that
    finishes in the call that brings its last piece plans that piece as its end.  Round r of a
    call runs the r-th piece of every stream that has one (or the last segment of a stream that
    finishes with no samples) as packs of at most max_samples samples; a pack is one packed
    forward whose launches do not depend on how many streams it holds (DESIGN.md section 16).
    This is the one windowed engine: a FeatureStream is a one-stream pool, and extract_long one
    push of a whole recording into one.  Between calls the device holds each stream's recent
    samples in a ring of an arena and its QRNN state in a (max_streams, H) table; the host holds
    four counters per stream."""

    def __init__(self, model, device, max_streams, window=None, max_samples=None):
        cfg = model.cfg
        win = _check_window(cfg, _enc.min_window(cfg) if window is None else window)
        if not 1 <= int(max_streams) <= 65535:           # one grid row per stream
            raise ValueError("max_streams must be in 1..65535, got %r" % (max_streams,))
        cap = STREAM_POOL_MAX_SAMPLES if max_samples is None else int(max_samples)
        if cap < 1:
            raise ValueError("max_samples must be positive, got %r" % (max_samples,))
        self.model, self.device, self.cfg = model, device, cfg
        self.max_streams, self.max_samples = int(max_streams), cap
        self.chunk = _enc.stream_chunk(cfg, win)
        self.seg_cap = _enc.window_capacity(cfg, win)         # the longest segment
        self.capacity = max(cap, self.seg_cap)
        self.plan = model._packed_plan(self.capacity, device)
        self.ring_cap = _enc.stream_ring_capacity(cfg, win)
        self.ring = torch.zeros(self.max_streams * self.ring_cap, dtype=torch.float32,
                                device=device)
        self.state = (torch.zeros(self.max_streams * self.plan.H, dtype=torch.float32,
                                  device=device) if self.plan.rnn else None)
        self._free = list(range(self.max_streams - 1, -1, -1))
        self._streams, self._next_id = {}, 0
        # two host staging slots (samples, table, event) and their device copies
        self._pin = device.type == "cuda"
        self._host = [[None, None, None], [None, None, None]]
        self._hi = 0
        self._stage = torch.empty(0, dtype=torch.float32, device=device)
        self._tab = torch.empty(0, dtype=torch.int32, device=device)

    def open(self):
        """A new stream's id; its slot starts from zero QRNN state and no samples."""
        if not self._free:
            raise RuntimeError("StreamPool: %d streams are open already (max_streams); finish "
                               "one first" % self.max_streams)
        sid, self._next_id = self._next_id, self._next_id + 1
        self._streams[sid] = _PoolStream(self._free.pop())
        return sid

    def __len__(self):
        return len(self._streams)

    def _release(self, sid):
        """Close stream sid (if open) and free its slot."""
        st = self._streams.pop(sid, None)
        if st is not None:
            self._free.append(st.slot)

    def push(self, blocks, finish=()):
        """blocks: {id: fp32 (T,), (1,T) or (1,1,T) samples on the CPU or the pool's GPU};
        finish: ids whose recording ends after this call's samples.  -> {id: (1, emb, n)} for
        every id in either, views of one buffer.  Every argument is checked, and every segment
        planned, before the first launch: a call that raises changes no stream."""
        return self._push(blocks, finish, None)

    def _push(self, blocks, finish, out, state_log=None):
        """push(), writing the frames into `out` (None: a new buffer) as consecutive (emb, n)
        blocks, one per id in the order of blocks then finish.  state_log (WaveFe.encode_long):
        an iterator over zeroed (H,) device rows; the QRNN state entering each segment, in the
        order the segments run, is copied into the next one (a stream's first segment starts
        from zero and leaves its row as it is)."""
        m, emb = self.model, self.model.emb_dim
        if m.training:
            raise RuntimeError("WaveFe.streams runs the encoder in eval mode; call .eval() first")
        if m.W.weight.device != self.device:
            raise RuntimeError("pase_b200.WaveFe runs on CUDA (sm_90a) only; the module lives "
                               "on %s, the pool on %s. There is no CPU path."
                               % (m.W.weight.device, self.device))
        if not isinstance(blocks, dict):
            raise TypeError("blocks must map stream ids to sample tensors, got %s"
                            % type(blocks).__name__)
        fin = list(dict.fromkeys(finish))
        ids = list(blocks) + [i for i in fin if i not in blocks]
        for i in ids:
            if i not in self._streams:
                raise KeyError("StreamPool: stream %r is unknown or finished" % (i,))
        xs = {}
        for i, b in blocks.items():
            try:
                x = _recording(b)
            except (TypeError, ValueError) as e:
                raise type(e)("stream %r: %s" % (i, e)) from None
            if x.device.type != "cpu" and x.device != self.device:
                raise ValueError("stream %r: samples on %s, the pool runs on %s"
                                 % (i, x.device, self.device))
            xs[i] = x
        steps, new = self._plan(ids, xs, set(fin))
        # the plan of the model's LRU, not one this pool pinned when the LRU has moved on
        self.plan = m._packed_plan(self.capacity, self.device)

        col, views, ocol = 0, {}, {}
        total = sum(new[i][1] - self._streams[i].done for i in ids)
        if out is None:
            out = torch.empty(emb * total, dtype=torch.float32, device=self.device)
        out = out.view(-1)
        for i in ids:
            nf = new[i][1] - self._streams[i].done
            views[i] = out[col * emb:(col + nf) * emb].view(1, emb, nf)
            ocol[i] = col
            col += nf
        if total:
            m._sinc_consts(self.device)
        params = dict(m.named_parameters())
        with torch.no_grad():
            for r in range(max((len(s) for s in steps.values()), default=0)):
                entries = [(i, steps[i][r]) for i in ids if r < len(steps[i])]
                self._round(entries, out, ocol, new, params, state_log)
        for i in ids:                                  # commit
            self._streams[i].n, self._streams[i].done, self._streams[i].keep = new[i]
        for i in fin:
            self._release(i)
        return views

    def _plan(self, ids, xs, fin):
        """Every stream's steps of this call on the host, through encoder.stream_step: per id a
        list of (piece or None, n before it, done before it, keep before it, segment or None)
        and its counters after the call.  A finishing stream's last piece is planned at_end (a
        finish with no samples is a step of its own).  Raises before any launch."""
        cfg, steps, new = self.cfg, {}, {}
        for i in ids:
            st = self._streams[i]
            n, done, keep = st.n, st.done, st.keep
            x = xs.get(i)
            L = 0 if x is None else x.numel()
            pieces = [x[a:a + self.chunk] for a in range(0, L, self.chunk)]
            if i in fin and not pieces:
                pieces = [None]
            out = []
            for k, piece in enumerate(pieces):
                end = i in fin and k + 1 == len(pieces)
                try:
                    n1, d1, k1, seg = _enc.stream_step(cfg, n, done, keep,
                                                       0 if piece is None else piece.numel(), end)
                except (ValueError, NotImplementedError) as e:
                    raise type(e)("stream %r: %s" % (i, e)) from None
                if n1 - keep > self.ring_cap or (seg is not None and (
                        seg["seg_start"] < keep or seg["seg_len"] > self.seg_cap)):
                    raise RuntimeError("StreamPool: stream %r would read samples %d .. %d from a "
                                       "ring of %d" % (i, keep, n1, self.ring_cap))
                if piece is not None or seg is not None:
                    out.append((piece, n, done, keep, seg))
                n, done, keep = n1, d1, k1
            steps[i], new[i] = out, (n, done, keep)
        return steps, new

    def _round(self, entries, out, ocol, new, params, state_log=None):
        """One round: stage the new samples, upload one table for every pack, then per pack the
        gather, the packed front end, the carried scan, the output projection and the place."""
        cfg, plan, emb = self.cfg, self.plan, self.model.emb_dim
        call = _ops.call
        # staging: host pieces first (one copy through pinned memory), then device pieces
        host_p = [(i, e[0]) for i, e in entries if e[0] is not None and
                  not (self._pin and e[0].is_cuda)]
        dev_p = [(i, e[0]) for i, e in entries if e[0] is not None and self._pin and e[0].is_cuda]
        stage_off, a = {}, 0
        for i, p in host_p + dev_p:
            stage_off[i] = a
            a += p.numel()
        nh = sum(p.numel() for _, p in host_p)
        # packs over the round's segments; rows that only append go with the first pack
        segs = [(i, e) for i, e in entries if e[4] is not None]
        appends = [(i, e) for i, e in entries if e[4] is None and e[0] is not None]
        lengths = [e[4]["seg_len"] for _, e in segs]
        packs = _enc.split_packs(lengths, self.max_samples) or [(0, 0)]
        fold = plan.precision.sinc_fold
        geoms = _enc.utterance_geometry(cfg, lengths, fold)
        parts, jobs, off = [], [], 0
        for p, (a0, b0) in enumerate(packs):
            g_rows, c_rows, p_rows = [], [], []
            pk = segs[a0:b0]
            if pk:
                host, sec, sz = _enc.packed_layout(plan, lengths[a0:b0], geoms[a0:b0], None)
                q0 = np.concatenate([[0], np.cumsum(sz["Tq"])])
                wave_off = 0
            for k, (i, (piece, n0, d0, k0, seg)) in enumerate(pk):
                slot = self._streams[i].slot
                s, sl = seg["seg_start"], seg["seg_len"]
                nn = 0 if piece is None else piece.numel()
                g_rows.append([slot, n0 % self.ring_cap, nn, stage_off.get(i, 0),
                               s % self.ring_cap, n0 - s, sl, wave_off])
                wave_off += sl
                r0 = int(q0[k]) + seg["crop_f0"]
                c_rows.append([r0, seg["crop_n"], slot, int(d0 == 0)])
                p_rows.append([r0, seg["crop_n"], ocol[i], new[i][1] - self._streams[i].done,
                               d0 - self._streams[i].done])
            if p == 0:
                for i, (piece, n0, _, _, _) in appends:
                    g_rows.append([self._streams[i].slot, n0 % self.ring_cap, piece.numel(),
                                   stage_off[i], 0, 0, 0, 0])
            if not g_rows:
                continue
            job = dict(segs=len(pk), gather=(off, len(g_rows)),
                       entering=[(self._streams[i].slot, e[2]) for i, e in pk])
            parts.append(np.asarray(g_rows, dtype=np.int64).reshape(-1))
            off += parts[-1].size
            job["max_len"] = max(max(r[2], r[6]) for r in g_rows)
            if pk:
                job["sec"] = {k: v + off for k, v in sec.items()}
                job["sz"] = sz
                parts.append(host.numpy().astype(np.int64))
                off += parts[-1].size
                job["carry"] = off
                parts.append(np.asarray(c_rows, dtype=np.int64).reshape(-1))
                off += parts[-1].size
                job["place"] = off
                job["max_T"] = max(r[1] for r in p_rows)
                parts.append(np.asarray(p_rows, dtype=np.int64).reshape(-1))
                off += parts[-1].size
            jobs.append(job)
        if not jobs:
            return
        table = np.concatenate(parts)
        assert np.abs(table).max() < _enc.INDEX_LIMIT     # `old` may be negative
        stage, tab = self._upload([p for _, p in host_p], nh, a, table)
        if dev_p:                                       # device blocks: one launch
            torch.cat([p for _, p in dev_p], out=stage[nh:a])

        bo = plan.bn_out
        for job in jobs:
            g0, gn = job["gather"]
            call("pase_stream_gather", stage, self.ring, self.ring_cap, plan.wave, tab[g0:], gn,
                 job["max_len"])
            if not job["segs"]:
                continue
            sz, sec = job["sz"], job["sec"]
            _enc._packed_front_launch(plan, self.model, plan.wave, sz,
                                      lambda name, sec=sec: tab[sec[name]:], params)
            if plan.rnn:
                if state_log is not None:
                    H = plan.H
                    for slot, d0 in job["entering"]:
                        row = next(state_log)
                        if d0 > 0:
                            row.copy_(self.state[slot * H:(slot + 1) * H])
                call("pase_qrnn_scan_fwd_carry_var", plan.Yg, plan.cat, plan.Kc, plan.Cst,
                     self.state, tab[job["carry"]:], job["segs"], plan.H)
            _enc._out_proj(plan, self.model, params, sz["rows"])
            call("pase_out_place_var", plan.yout, bo[2], bo[3], out, tab[job["place"]:],
                 job["segs"], job["max_T"], emb)

    def _upload(self, host_pieces, nh, n, table):
        """The round's samples (host pieces into staging[0:nh]) and its table, each with one
        copy from a pinned slot; the host waits only when it reuses a slot whose copies have
        not finished.  -> (device staging, device table); both grow, never shrink."""
        if self._stage.numel() < n:
            self._stage = torch.empty(_grow(n), dtype=torch.float32, device=self.device)
        if self._tab.numel() < table.size:
            self._tab = torch.empty(_grow(table.size), dtype=torch.int32, device=self.device)
        slot, self._hi = self._host[self._hi], self._hi ^ 1
        if slot[2] is not None:
            slot[2].synchronize()               # this slot's last copies have finished
        if slot[0] is None or slot[0].numel() < nh:
            slot[0] = _host_buffer(_grow(nh), torch.float32, self._pin)
        if slot[1] is None or slot[1].numel() < table.size:
            slot[1] = _host_buffer(_grow(table.size), torch.int32, self._pin)
        if nh:
            torch.cat(host_pieces, out=slot[0][:nh])
            self._stage[:nh].copy_(slot[0][:nh], non_blocking=True)
        slot[1][:table.size].copy_(torch.from_numpy(table.astype(np.int32)))
        self._tab[:table.size].copy_(slot[1][:table.size], non_blocking=True)
        if self._pin:
            slot[2] = torch.cuda.Event()
            slot[2].record()
        return self._stage, self._tab


def _grow(n):
    """Capacity for n elements: the next power of two (at least 1024)."""
    return max(1024, 1 << (int(n) - 1).bit_length())


def _host_buffer(n, dtype, pinned):
    t = torch.empty(n, dtype=dtype)
    return t.pin_memory() if pinned else t
