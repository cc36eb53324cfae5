"""Worker heads ("minions") of PASE/PASE+ over the C-ABI kernels: drop-in for
pase/models/Minions/minions.py (MLPMinion 452-528, DecoderMinion 365-449,
SPCMinion 575-649) and cls_minions.py (LIM 53-74, GIM 76-99, SPC 101-115).

Constructor kwargs, attribute names (``name``, ``loss``, ``loss_weight``), the
``forward(x, alpha=1, device=None)`` protocol and the state_dict keys
(``blocks.i.W.*``, ``blocks.i.act.weight``, ``blocks.i.deconv.*``, ``W.*``,
``minion.*``) are the reference's.  Internally activations are channel-last rows;
``forward`` accepts either the reference's (B,C,T) tensors or rows tagged by the
encoder, and returns a (B, F, T)-shaped view of its channel-last output.
"""
import json
import random

import torch
import torch.nn as nn

from .modules import Model
from . import functional as Fn
from . import decoder as _dec


def _unsupported(cond, what):
    if cond:
        raise NotImplementedError("pase_b200 minion: %s is not implemented natively" % what)


class RowsInput(object):
    """Channel-last activation handed between the encoder and the heads."""

    def __init__(self, rows, B, T):
        self.rows, self.B, self.T = rows, B, T          # rows: (B*T, C) tensor

    @staticmethod
    def of(x):
        if isinstance(x, RowsInput):
            return x
        tag = getattr(x, "_pase_rows_in", None)
        if tag is not None:
            return tag
        assert x.dim() == 3, "expected a (B,C,T) tensor"
        return RowsInput(Fn.nct_to_rows(x), x.shape[0], x.shape[2])


def rows_to_pred(rows, B, T, ncols):
    """(B*T, >=ncols) rows (row stride ld) -> reference-shaped (B, ncols, T) view, tagged with
    its buffer."""
    ld = rows.stride(0) if rows.shape[0] > 1 else rows.shape[1]
    pred = torch.as_strided(rows, (B, ncols, T), (T * ld, 1, ld), rows.storage_offset())
    pred._pase_rows = (rows, ncols)
    return pred


class _MLPBlockParams(nn.Module):
    """Parameter container with MLPBlock's names (modules.py:527-556)."""

    def __init__(self, ninp, fmaps):
        super().__init__()
        self.W = nn.Conv1d(ninp, fmaps, 1)
        self.act = nn.PReLU(fmaps)


class MLPMinion(Model):
    def __init__(self, num_inputs, num_outputs, dropout, dropout_time=0.0, hidden_size=256,
                 dropin=0.0, hidden_layers=2, context=1, tie_context_weights=False, skip=True,
                 loss=None, loss_weight=1., keys=None, augment=False, r=1, name='MLPMinion',
                 ratio_fixed=None, range_fixed=None, dropin_mode='std', drop_channels=False,
                 emb_size=100):
        super().__init__(name=name)
        _unsupported(context != 1, "context > 1")
        _unsupported(dropout != 0 or dropin != 0 or dropout_time != 0, "dropout")
        _unsupported(tie_context_weights, "tie_context_weights")
        _unsupported(num_inputs % 4 != 0 or hidden_size % 4 != 0, "channel counts not multiple of 4")
        self.num_inputs, self.context, self.skip = num_inputs, context, skip
        self.hidden_size, self.hidden_layers = hidden_size, hidden_layers
        self.loss, self.loss_weight, self.keys = loss, loss_weight, keys
        self.r = r
        self.num_outputs = num_outputs * r
        self.blocks = nn.ModuleList()
        ninp = num_inputs
        for _ in range(hidden_layers):
            self.blocks.append(_MLPBlockParams(ninp, hidden_size))
            ninp = hidden_size
        self.W = nn.Conv1d(ninp, self.num_outputs, 1)

    def forward_rows(self, rows):
        h = rows
        for blk in self.blocks:
            C = blk.W.weight.shape[0]
            u = Fn.linear_rows(h, blk.W.weight, blk.W.bias)
            h = Fn.prelu_rows(u, blk.act.weight, C)[:, :C]      # drop the leading-dim padding
        return Fn.linear_rows(h, self.W.weight, self.W.bias), h

    def forward(self, x, alpha=1, device=None, label=None):
        """label (optional, (B, F, T)): fuse the output layer with the worker's contextualised
        MSE (``pase.fuse_regression_loss``): the returned "prediction" is then a zero-stride
        placeholder of the reference shape that carries the already-reduced loss
        (``ContextualizedLoss`` returns it); the (B, F*r, T) prediction is never stored."""
        xin = RowsInput.of(x)
        if label is not None and not self.skip and self._can_fuse(xin, label):
            h = xin.rows
            for blk in self.blocks:
                C = blk.W.weight.shape[0]
                h = Fn.prelu_rows(Fn.linear_rows(h, blk.W.weight, blk.W.bias), blk.act.weight, C)[:, :C]
            F = label.shape[1]
            loss = Fn.fused_linear_ctx_mse(h, self.W.weight, self.W.bias, label.to(h.device), F,
                                           int(self.r))
            pred = torch.zeros(1, device=h.device).expand(xin.B, self.num_outputs, xin.T)
            pred._pase_fused_loss = loss
            return pred
        y, h = self.forward_rows(xin.rows)
        pred = rows_to_pred(y, xin.B, xin.T, self.num_outputs)
        if self.skip:
            return pred, rows_to_pred(h, xin.B, xin.T, self.hidden_size)
        return pred

    def _can_fuse(self, xin, label):
        loss = self.loss
        if getattr(loss, "kind", None) != "MSELoss" or not self.r or int(self.r) % 2 != 1:
            return False
        if label.dim() != 3 or label.shape[1] * int(self.r) != self.num_outputs or \
                label.shape[0] != xin.B or label.shape[2] != xin.T:
            return False
        K = self.W.weight.shape[1]
        return Fn.fused_head_ok(K, K if self.blocks else xin.rows.stride(0))


class SPCMinion(MLPMinion):
    """Future-vs-past frame discrimination (minions.py:575-649).  The three frames are drawn
    from Python's ``random`` exactly like the reference (host RNG, three draws per call), unless
    ``frame_table`` holds a device int64 tensor {t, future_t, past_t}: a captured training step
    (``pase_b200.graph.GraphedTrainStep``) sets it to its own table, which its planner fills with
    ``draw_frames`` before every replay."""

    def __init__(self, num_inputs, num_outputs, dropout, hidden_size=256, hidden_layers=2,
                 ctxt_frames=5, seq_pad=16, skip=True, loss=None, loss_weight=1., keys=None,
                 name='SPCMinion'):
        super().__init__(num_inputs=(ctxt_frames + 1) * num_inputs, num_outputs=num_outputs,
                         dropout=dropout, hidden_size=hidden_size, hidden_layers=hidden_layers,
                         skip=skip, loss=loss, loss_weight=loss_weight, keys=keys, name=name)
        self.ctxt_frames, self.seq_pad = ctxt_frames, seq_pad
        self.frame_table = None

    def frames_ok(self, T):
        """Whether T frames leave the current frame's range [M + 1, T - M) non-empty (then the
        future and past ranges are non-empty too)."""
        M = self.seq_pad + self.ctxt_frames
        return T - M > M + 1

    def draw_frames(self, T, py=random):
        """(t, future_t, past_t) for T frames: the reference's three draws from `py`."""
        N, sp = self.ctxt_frames, self.seq_pad
        M = sp + N
        if not self.frames_ok(T):
            raise ValueError("SPCMinion %s: T'=%d frames leave range(%d, %d) for the current "
                             "frame empty (ctxt_frames=%d, seq_pad=%d)" % (self.name, T, M + 1,
                                                                           T - M, N, sp))
        t = py.choice(list(range(M + 1, T - M)))
        future_t = py.choice(list(range(t + sp, T - N)))
        past_t = py.choice(list(range(N, t - sp)))
        return t, future_t, past_t

    def forward(self, x, alpha=1, device=None):
        xin = RowsInput.of(x)
        B, T = xin.B, xin.T
        frames = self.frame_table if self.frame_table is not None else self.draw_frames(T)
        # reference flattens (B,C,N) channel-major: index c*N + n
        rows = Fn.spc_gather(xin.rows, B, T, self.ctxt_frames, self.seq_pad, frames)
        y, h = self.forward_rows(rows)
        pred = rows_to_pred(y, 2 * B, 1, self.num_outputs)
        if self.skip:
            return pred, rows_to_pred(h, 2 * B, 1, self.hidden_size)
        return pred


class _GDeconvParams(nn.Module):
    """Parameter container with GDeconv1DBlock's names (modules.py:558-589)."""

    def __init__(self, ninp, fmaps, kwidth, stride):
        super().__init__()
        pad = max(0, (stride - kwidth) // -2)
        self.deconv = nn.ConvTranspose1d(ninp, fmaps, kwidth, stride=stride, padding=pad)
        self.act = nn.PReLU(fmaps, init=0)
        self.kwidth, self.stride, self.pad = kwidth, stride, pad


class DecoderMinion(Model):
    """Waveform decoder worker: transposed-conv stack + MLP (minions.py:365-449)."""

    def __init__(self, num_inputs, num_outputs, dropout, dropout_time=0.0, shuffle=False,
                 shuffle_depth=7, hidden_size=256, hidden_layers=2,
                 fmaps=[256, 256, 128, 128, 128, 64, 64], strides=[2, 2, 2, 2, 2, 5],
                 kwidths=[2, 2, 2, 2, 2, 5], norm_type=None, skip=False, loss=None,
                 loss_weight=1., keys=None, name='DecoderMinion'):
        super().__init__(name=name)
        _unsupported(dropout != 0 or dropout_time != 0, "dropout")
        _unsupported(shuffle, "shuffle")
        _unsupported(norm_type is not None, "norm_type=%r" % norm_type)
        _unsupported(skip, "skip=True")
        self.num_inputs, self.num_outputs = num_inputs, num_outputs
        self.hidden_size, self.hidden_layers = hidden_size, hidden_layers
        self.fmaps, self.strides, self.kwidths = fmaps, strides, kwidths
        self.loss, self.loss_weight, self.keys, self.skip = loss, loss_weight, keys, skip
        self.blocks = nn.ModuleList()
        ninp = num_inputs
        self.n_deconv = 0
        for fmap, kw, stride in zip(fmaps, kwidths, strides):
            _unsupported((stride % 2) != (kw % 2), "transposed conv with odd/even trim")
            _unsupported(fmap % 4 != 0, "channel counts not multiple of 4")
            self.blocks.append(_GDeconvParams(ninp, fmap, kw, stride))
            ninp = fmap
            self.n_deconv += 1
        for _ in range(hidden_layers):
            self.blocks.append(_MLPBlockParams(ninp, hidden_size))
            ninp = hidden_size
        self.W = nn.Conv1d(hidden_size, num_outputs, 1)
        self._plans = {}

    def forward(self, x, alpha=1, device=None):
        xin = RowsInput.of(x)
        h, L = _dec.decoder_stack(self, xin.rows, xin.B, xin.T)       # (B*L, C) rows
        for blk in self.blocks[self.n_deconv:]:
            C = blk.W.weight.shape[0]
            u = Fn.linear_rows(h, blk.W.weight, blk.W.bias)
            h = Fn.prelu_rows(u, blk.act.weight, C)[:, :C]
        y = Fn.linear_rows(h, self.W.weight, self.W.bias)
        return rows_to_pred(y, xin.B, L, self.num_outputs)


def minion_maker(cfg):
    """cfg dict (or JSON path) -> minion (minions.py:11-35).  wavernn / gap / gru /
    regularizer workers are not part of workers.cfg / workers+.cfg and are out of scope."""
    if isinstance(cfg, str):
        with open(cfg, "r") as f:
            cfg = json.load(f)
    cfg = dict(cfg)
    mtype = cfg.pop('type', 'mlp')
    cfg.pop('transform', None)
    if mtype == 'mlp':
        return MLPMinion(**cfg)
    if mtype == 'decoder':
        return DecoderMinion(**cfg)
    if mtype == 'spc':
        return SPCMinion(**cfg)
    raise TypeError('Unrecognized minion type {}'.format(mtype))


# ------------------------------------------------ contrastive wrappers ------
def _pair_labels(pred, device):
    """[ones; zeros] with the prediction's shape (make_labels, cls_minions.py:47-51)."""
    half = pred.shape[0] // 2
    lab = torch.cat([torch.ones(half, 1, pred.shape[2], device=device),
                     torch.zeros(half, 1, pred.shape[2], device=device)], 0)
    lab._pase_pairs = half * pred.shape[2]
    return lab


def _pair_rows(h, augment):
    """h: three RowsInput (chunk, ctxt, rand) -> rows of [pos; neg] pairs, channels
    concatenated (make_samples, cls_minions.py:29-43)."""
    a, b, c = (RowsInput.of(t) for t in h)
    pos = [torch.cat([a.rows, b.rows], 1)]
    neg = [torch.cat([a.rows, c.rows], 1)]
    if augment:
        pos.append(torch.cat([b.rows, a.rows], 1))
        neg.append(torch.cat([b.rows, c.rows], 1))
    rows = torch.cat(pos + neg, 0)
    return rows, a.B * (2 if augment else 1) * 2, a.T


class _PairWorker(Model):
    def __init__(self, cfg, emb_dim, num_inputs):
        super().__init__(name=cfg['name'])
        cfg = dict(cfg)
        cfg['num_inputs'] = num_inputs
        self.augment = bool(cfg.get('augment', False))
        self.minion = minion_maker(cfg)
        self.loss = self.minion.loss
        self.loss_weight = self.minion.loss_weight


class LIM(_PairWorker):
    """Local info-max: per-frame (chunk,ctxt) vs (chunk,rand) discrimination."""

    def __init__(self, cfg, emb_dim):
        super().__init__(cfg, emb_dim, 2 * emb_dim)

    def forward(self, x, alpha=1, device=None):
        rows, nb, T = _pair_rows(x, self.augment)
        y = self.minion(RowsInput(rows, nb, T), alpha)
        y = y[0] if isinstance(y, tuple) else y
        return y, _pair_labels(y, rows.device)


class GIM(_PairWorker):
    """Global info-max: time-averaged pairs."""

    def __init__(self, cfg, emb_dim):
        super().__init__(cfg, emb_dim, 2 * emb_dim)

    def forward(self, x, alpha=1, device=None):
        rows, nb, T = _pair_rows(x, self.augment)
        rows = Fn.time_mean_rows(rows, nb, T)
        y = self.minion(RowsInput(rows, nb, 1), alpha)
        y = y[0] if isinstance(y, tuple) else y
        return y, _pair_labels(y, rows.device)


class SPC(_PairWorker):
    def __init__(self, cfg, emb_dim):
        super().__init__(cfg, emb_dim, emb_dim)

    def forward(self, x, alpha=1, device=None):
        y = self.minion(x, alpha)
        y = y[0] if isinstance(y, tuple) else y
        return y, _pair_labels(y, y.device)


def cls_worker_maker(cfg, emb_dim):
    name = cfg["name"]
    if name == "mi":
        return LIM(cfg, emb_dim)
    if name == "cmi":
        return GIM(cfg, emb_dim)
    if name == "spc":
        return SPC(cfg, emb_dim)
    if name == "gap":
        raise NotImplementedError("gap worker is not part of workers.cfg / workers+.cfg")
    return minion_maker(cfg)
