"""H100-native WaveFe encoder engine: geometry, HBM buffer plan and the
forward/backward orchestration over the C-ABI kernels.

Formulation (DESIGN.md section 3).  Activations are channel-last (n, t, c).
Every strided 1-D convolution of the reference (FeBlock, modules.py:1058-1077;
SincConv_fast, modules.py:920-934) becomes ONE GEMM whose A operand is an
*overlapping-row view* of the reflect-padded activation: row (n, t) is the
k*Cin contiguous floats starting at time t*stride, so no im2col is ever
materialised and all strides (1, 2, 10) use the same kernel.  The 251-tap
Cin=1 sinc layer is folded 4x in time (polyphase) so that it has the same
shape.  Train-mode BatchNorm statistics are accumulated in the GEMM epilogue;
BN+PReLU+reflect-pad+dense-skip pooling are one elementwise pass that writes
the next layer's padded operand.  Dense skips are pooled BEFORE their 1x1
projection (mean-pool commutes with a bias-free 1x1 conv, frontend.py:182,
213-232), which removes the reference's (N,256,T) intermediates; the pooled
skips and the QRNN output are concatenated so W + all skips are one GEMM.
"""
import math

import numpy as np
import torch

from . import gemm, ops

BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def _cdiv(a, b):
    return -(-a // b)


def _ru(a, m):
    return _cdiv(a, m) * m


def conv_pads(k, stride, sinc):
    """Reflect pad (left, right): SincConv_fast modules.py:922-928, FeBlock
    modules.py:1058-1071 (dilation 1)."""
    if sinc:
        return (k // 2 - 1, k // 2) if stride > 1 else (k // 2, k // 2)
    if k <= 1:
        return (0, 0)
    if stride > 1 or k % 2 == 0:
        return (k // 2 - 1, k // 2)
    return (k // 2, k // 2)


class ConvGeom(object):
    """Static geometry of one encoder block for a given input length."""

    def __init__(self, idx, sinc, Cin, Cout, k, s, L_in, sinc_fold=4):
        self.idx, self.sinc = idx, sinc
        self.Cin, self.Cout, self.k, self.s, self.L_in = Cin, Cout, k, s, L_in
        self.padL, self.padR = conv_pads(k, s, sinc)
        if self.padL >= L_in or self.padR >= L_in:
            raise ValueError("block %d: reflect pad (%d,%d) needs an input longer than "
                             "%d samples" % (idx, self.padL, self.padR, L_in))
        self.Tpad = L_in + self.padL + self.padR
        self.T_out = (self.Tpad - k) // s + 1
        if sinc:
            # polyphase fold: row u of the GEMM produces times fold*u .. fold*u+fold-1
            self.fold = sinc_fold
            self.lda = sinc_fold                       # floats between consecutive rows
            self.K = _ru(k + sinc_fold - 1, sinc_fold if sinc_fold >= 32 else 4)
            self.Nn = sinc_fold * Cout
            self.P = _cdiv(self.Tpad, sinc_fold)       # rows per sample
            self.rows_out = _cdiv(self.T_out, sinc_fold)
            # input gradient (DESIGN.md section 17): row v of the transposed convolution gives
            # the padded positions fold*v .. fold*v+fold-1 from the dg_rows folded rows of dy
            # that start dg_halo frames earlier
            self.dg_halo = _cdiv(k - 1, sinc_fold) * sinc_fold
            self.dg_rows = self.dg_halo // sinc_fold + 1
            self.dg_K = self.dg_rows * sinc_fold * Cout
            self.dg_P = self.P + self.dg_rows - 1      # rows per sample of the haloed dy copy
        else:
            self.fold = 1
            self.lda = s * Cin
            self.K = k * Cin
            self.Nn = Cout
            self.P = _cdiv(self.Tpad, s)
            self.rows_out = self.T_out
        self.Ty = self.rows_out * self.fold            # time pitch of the raw output
        self.apad_floats = self.P * self.lda           # per sample
        # backward-data: taps of the polyphase transposed convolution
        self.taps = _cdiv(k, s)
        self.Pd = self.P + self.taps - 1               # rows per sample of zero-padded dy

    @property
    def count(self):
        return self.T_out


def build_geometry(cfg, T, sinc_fold=4):
    geoms, L, cin = [], T, cfg["num_inputs"]
    for i, (k, s, f) in enumerate(zip(cfg["kwidths"], cfg["strides"], cfg["fmaps"])):
        sinc = bool(cfg["sincnet"]) and i == 0
        if sinc and k % 2 == 0:
            k += 1                                     # modules.py:835-836
        g = ConvGeom(i, sinc, cin, f, k, s, L, sinc_fold)
        geoms.append(g)
        L, cin = g.T_out, f
    return geoms


def frame_counts(cfg, T):
    return [g.T_out for g in build_geometry(cfg, T)]


class EncoderPlan(object):
    """All HBM buffers of one (N, T) problem, allocated once and reused every
    step (180 GB HBM: nothing is recomputed or re-allocated).  Padded operand
    buffers are zero-initialised once; kernels only ever write their valid
    region, so halos / slack stay finite.

    Storage by precision (DESIGN.md section 3):
      fp32 / tf32 / 3xtf32: everything fp32 (3xtf32 adds tf32-residual twins of the operands);
      bf16 : GEMM operands, raw conv outputs y, gradients dxpad / du / dy in bf16; statistics,
             weights' master copies, weight gradients and the small output-side tensors fp32;
      3xf16: GEMM operands as fp16 (hi, lo') pairs, everything else fp32."""

    def __init__(self, cfg, N, T, device, prec="fp32"):
        self.N, self.T = N, T
        self._setup(cfg, device, prec, lambda fold: build_geometry(cfg, T, fold))
        G = self.geoms
        self.Tq = G[-1].T_out
        self.pool_d = [max(g.T_out // self.Tq, 1) for g in G[:-1]]
        self.rows = N * self.Tq
        self._alloc([N * g.apad_floats for g in G], [N * g.rows_out * g.Nn for g in G],
                    self.rows, N * (self.Tq + 1))

    def _setup(self, cfg, device, prec, geometry):
        """Length-independent state: precision, layer shapes (geometry(sinc_fold) -> geoms),
        column layout of the output projection's operand."""
        self.cfg, self.device = cfg, device
        if prec not in gemm.PRECISIONS:
            raise ValueError("precision must be one of %s" % (sorted(gemm.PRECISIONS),))
        self.precision = p = gemm.PRECISIONS[prec]
        self._ops = {}             # name -> gemm.Operand
        self._wtables = {}
        self.geoms = geometry(p.sinc_fold)
        G = self.geoms
        if p.esz == 2:
            for g in G:
                if (g.lda % p.eb) or (g.Cout % p.eb and not g.sinc):
                    raise NotImplementedError(
                        "precision %r needs channel counts that are multiples of %d (block %d: "
                        "Cin=%d Cout=%d stride=%d)" % (prec, p.eb, g.idx, g.Cin, g.Cout, g.s))
        self.nblk = len(G)
        self.emb = cfg["emb_dim"]
        self.rnn = bool(cfg["rnn_pool"])
        self.skips = bool(cfg["denseskips"])
        self.norm_out = bool(cfg["norm_out"])
        self.Clast = G[-1].Cout
        self.H = (cfg["rnn_dim"] // 2) * 2 if self.rnn else 0
        # concatenated [rnn-out | pooled skips] operand of the output projection
        self.col_off = []
        off = self.H if self.rnn else self.Clast
        for g in G[:-1]:
            self.col_off.append(off)
            if self.skips:
                off += g.Cout
        self.Kc = off

    def _alloc(self, n_apad, n_y, rows, xq_rows):
        """Forward buffers: padded operands of n_apad[l] elements (+ slack), raw conv outputs of
        n_y[l], `rows` output frames, `xq_rows` rows of the QRNN input."""
        G, p, device = self.geoms, self.precision, self.device
        f32 = dict(dtype=torch.float32, device=device)
        f64 = dict(dtype=torch.float64, device=device)
        opd = dict(dtype=p.dtype, device=device)
        yd = dict(dtype=torch.bfloat16 if p.act_bf16 else torch.float32, device=device)
        z = lambda n: torch.zeros(int(n), **f32)
        e = lambda n: torch.empty(int(n), **f32)
        zo = lambda n: torch.zeros(int(n), **opd)          # operand-format buffers (hi / lo)
        zlo = lambda n: torch.zeros(int(n), **opd) if p.split else None

        self.apad, self.apad_lo, self.y, self.bn = [], [], [], []
        self.Wt = []
        for g, na, ny in zip(G, n_apad, n_y):
            n_apad = na + g.K + 64
            self.apad.append(zo(n_apad))
            self.apad_lo.append(zlo(n_apad))
            self._ops[("apad", g.idx)] = gemm.Operand(self.apad[-1], self.apad_lo[-1])
            self.y.append(torch.empty(int(ny), **yd))
            self.bn.append(torch.zeros(4, g.Cout, **f32))       # mean, invstd, scale, shift
            self.Wt.append(e(g.Nn * g.K))
        if self.rnn:
            Cq, H = self.Clast, self.H
            n_xq = xq_rows * Cq + 2 * Cq + 64
            self.xq, self.xq_lo = zo(n_xq), zlo(n_xq)
            self._ops["xq"] = gemm.Operand(self.xq, self.xq_lo)
            self.Yg, self.Cst = e(rows * 3 * H), e(rows * H)
            self.Wq = e(3 * H * 2 * Cq)
        self.cat = z(rows * self.Kc)
        self.Wcat = e(self.emb * self.Kc)
        self.yout = e(rows * self.emb)
        self.bn_out = torch.zeros(4, self.emb, **f32)
        self.bn_out[1].fill_(1.0)
        self.bn_out[2].fill_(1.0)

        # double-precision accumulators: forward batch statistics ...
        self.fs_off, n = [], 0
        for g in G:
            self.fs_off.append(n)
            n += 2 * g.Nn
        self.fs_out = n
        n += 2 * self.emb
        self.stats_f = torch.zeros(n, **f64)
        self.zeros64 = torch.zeros(max(2 * max(g.Cout for g in G), 2 * self.emb), **f64)
        # everything only the backward pass touches is allocated on first use
        # (`ensure_backward`): inference / feature extraction at a new (N, T) -- the main
        # downstream use, one plan per utterance length -- costs the forward buffers only
        self.backward_ready = False
        self.dWt = self.Wd = self.dyz = self.dyz_lo = self.dxpad = self.gscale = None
        self.dYg = self.dsrc = self.WqT = self.dWq = None
        self.dcat = self.WcatT = self.dWcat = self.g = None
        self.stats_b = self.grad_vec = self.amax = None
        self.dyh = self.dyh_lo = self.filt = self.Wdg = None     # ensure_input_grad
        self.generation = 0

    def ensure_backward(self):
        """Allocate the backward-only buffers (input / output gradients in operand format,
        weight-gradient and dgrad-weight layouts, fp64 reduction accumulators).  Called by
        WaveFe.encode before a forward that will be differentiated, i.e. during the eager
        warm-up steps and never inside a CUDA-graph capture."""
        if self.backward_ready:
            return
        N = self.N
        self._alloc_backward(
            [N * g.rows_out * g.Nn + 128 if g.sinc else N * g.Pd * g.Cout + g.taps * g.Cout + 128
             for g in self.geoms],
            [N * g.apad_floats for g in self.geoms], self.rows, self.rows)

    def _alloc_backward(self, n_dyz, n_dxpad, rows, yg_rows):
        """Backward buffers: each block's output gradient of n_dyz[l] elements in the GEMM
        format, its input gradient of n_dxpad[l] (blocks > 0), `rows` output frames and `yg_rows`
        rows of the QRNN gate gradients."""
        G, p, device = self.geoms, self.precision, self.device
        f32 = dict(dtype=torch.float32, device=device)
        f64 = dict(dtype=torch.float64, device=device)
        opd = dict(dtype=p.dtype, device=device)
        yd = dict(dtype=torch.bfloat16 if p.act_bf16 else torch.float32, device=device)
        z = lambda n: torch.zeros(int(n), **f32)
        e = lambda n: torch.empty(int(n), **f32)
        zo = lambda n: torch.zeros(int(n), **opd)
        zlo = lambda n: torch.zeros(int(n), **opd) if p.split else None
        f16x2 = p.fmt == gemm.FMT_F16X2           # gradients carry power-of-two scales
        self.dWt, self.Wd, self.dyz, self.dyz_lo, self.dxpad, self.gscale = [], [], [], [], [], []
        for g, nd, nx in zip(G, n_dyz, n_dxpad):
            self.dWt.append(e(g.Nn * g.K))
            gs = torch.ones(2, **f32) if f16x2 else None
            self.gscale.append(gs)
            if g.sinc:
                self.Wd.append(None)
                self.dxpad.append(None)
            else:
                self.Wd.append(e(g.s * g.Cin * g.taps * g.Cout))
                self.dxpad.append(torch.empty(int(nx), **yd) if g.idx > 0 else None)
            self.dyz.append(zo(nd))
            self.dyz_lo.append(zlo(nd))
            self._ops[("dyz", g.idx)] = gemm.Operand(self.dyz[-1], self.dyz_lo[-1], gs)
        if self.rnn:
            Cq, H = self.Clast, self.H
            self.dYg = z(yg_rows * 3 * H + 64)
            self.dsrc = e(yg_rows * 2 * Cq)
            self.WqT = e(2 * Cq * 3 * H)
            self.dWq = e(3 * H * 2 * Cq)
        self.dcat = e(rows * self.Kc)
        self.WcatT = e(self.Kc * self.emb)
        self.dWcat = e(self.emb * self.Kc)
        self.g = torch.zeros(rows * self.emb + 64, **f32)     # +slack: TC wgrad reads whole blocks
        # backward reductions: per block S1,S2,dalpha,dbias; output S1,S2; qrnn bias; W bias
        self.bs_off, n = [], 0
        for g in G:
            self.bs_off.append(n)
            n += 4 * g.Cout
        self.bs_out = n
        n += 2 * self.emb
        self.bs_bq = n
        n += 3 * self.H
        self.bs_bw = n
        n += self.emb
        self.stats_b = torch.zeros(n, **f64)
        self.grad_vec = torch.zeros(n, **f32)
        # running maxima for the 3xF16 gradient scales: 2 floats per use, zeroed per backward
        self.amax = torch.zeros(2 * (self.nblk + 4), **f32) if f16x2 else None
        self.backward_ready = True

    def ensure_input_grad(self):
        """Allocate the buffers of the sinc layer's input gradient (_sinc_input_grad) on the
        first backward that returns the waveform gradient: the haloed copy of dy in the GEMM
        format (zero halos and slack, written only inside), the band-pass bank, its banded
        dgrad operand and the padded-waveform gradient dxpad[0]."""
        self.ensure_backward()
        if self.dyh is not None:
            return
        g, N, p, device = self.geoms[0], self.N, self.precision, self.device
        n = N * g.dg_P * g.Nn + g.dg_rows * g.Nn + 128          # + slack: rows past the last
        self.dyh = torch.zeros(n, dtype=p.dtype, device=device)
        self.dyh_lo = torch.zeros(n, dtype=p.dtype, device=device) if p.split else None
        self._ops[("dyh", 0)] = gemm.Operand(self.dyh, self.dyh_lo, self.gscale[0])
        self.filt = torch.empty(g.Cout * g.k, dtype=torch.float32, device=device)
        self.Wdg = torch.empty(g.fold * g.dg_K, dtype=torch.float32, device=device)
        self.dxpad[0] = torch.empty(N * g.P * g.fold, dtype=torch.float32, device=device)

    # -- GEMM operands -----------------------------------------------------------------
    def operand(self, name, buf, fresh=True, kind="act", n=None):
        """Operand `name` in the plan's GEMM format (gemm.Operand).  Operands whose producer
        writes the GEMM format directly (apad, xq, dyz, the conv weights) are registered with
        no fp32 source; everything else is the fp32 tensor `buf` converted into buffers kept
        per name (`fresh=False` reuses this step's earlier conversion; `n`: convert only the
        first n elements)."""
        op = self._ops.get(name)
        if op is not None and op.src is None:
            return op
        if op is None or op.src.numel() != buf.numel() or op.src.data_ptr() != buf.data_ptr():
            op = gemm.operand_buffers(self.precision, buf.numel(), self.device, kind, buf,
                                      torch.zeros)
            self._ops[name] = op
            fresh = True
        n = buf.numel() if n is None else n
        return gemm.convert(self.precision, op, n, kind) if fresh else op

    def w_operand(self, name, buf):
        """(hi, lo) buffers of a weight operand written by pase_conv_w_batch itself."""
        if self.precision.reads_fp32:
            return None, None
        op = self._ops.get(name)
        if op is None:
            op = gemm.operand_buffers(self.precision, buf.numel(), self.device, "weight",
                                      new=torch.zeros)
            self._ops[name] = op
        return op.hi, op.lo

    def w_batch(self, op, jobs, dst_base=None, key=None):
        """One launch for the weight re-layouts of every conv block (pase_conv_w_batch).
        jobs: [(src, dst tensor | element offset, hi, lo, Cout, Cin, k, s, taps, count)].
        The device job table is rebuilt only when a pointer changed."""
        ptr = lambda t: 0 if t is None else (t if isinstance(t, int) else t.data_ptr())
        # shared-memory tiled kernels (ops 3..5) when every job fits their tile shapes
        tiled = all(Cout % 32 == 0 and Cin % 8 == 0 and (Cin + 1) * k <= 12000
                    and 32 * (8 * k + 1) <= 12000
                    for (_, _, _, _, Cout, Cin, k, _, _, _) in jobs)
        rows, start, blocks = [], 0, 0
        for (src, dst, hi, lo, Cout, Cin, k, sd, taps, count) in jobs:
            rows.append([ptr(src), ptr(dst), ptr(hi), ptr(lo), Cout, Cin, k, sd, taps, start,
                         count, blocks])
            start += count
            blocks += (Cout // 32) * (Cin // 8) if op == 1 else Cout
        key = op if key is None else key
        ent = self._wtables.get(key)
        if ent is None or ent[0] != rows:
            table = torch.tensor(rows, dtype=torch.int64).reshape(-1).to(self.device)
            ent = (rows, table)
            self._wtables[key] = ent
        fmt = self.precision.fmt
        if tiled:
            ops.call("pase_conv_w_batch", ent[1], len(rows), blocks, op + 3, dst_base, fmt)
        else:
            ops.call("pase_conv_w_batch", ent[1], len(rows), start, op, dst_base, fmt)

    def nt(self, an, A, lda, afresh, bn, B, ldb, bfresh, C, ldc, M, N, K, alpha, bias,
           rows_in, t_valid, rows_out, fold, cs, cq, acc, akind="act", a_n=None):
        """C = alpha * A B^T (+ bias) in the plan's precision (gemm.nt) over the operands
        `an` / `bn` of buffers A / B (a_n: convert only the first a_n elements of A)."""
        return gemm.nt(self.precision, A, lda, A.numel(), B, ldb, C, ldc, M, N, K, alpha, bias,
                       rows_in, t_valid, rows_out, fold, cs, cq, acc, akind,
                       lambda: self.operand(an, A, afresh, akind, a_n),
                       lambda: self.operand(bn, B, bfresh, "weight"))

    def nt_var(self, an, A, lda, bn, B, ldb, bfresh, C, ldc, M, N, K, bias, tab, n, fold,
               cs=None, cq=None):
        """gemm.nt_var over the packed operand `an` (written in the GEMM format by its
        producer) and the weight operand `bn`."""
        return gemm.nt_var(self.precision, A, lda, A.numel(), B, ldb, C, ldc, M, N, K, bias, tab,
                           n, fold, lambda: self.operand(an, A, False),
                           lambda: self.operand(bn, B, bfresh, "weight"), cs, cq)

    def tn(self, an, A, lda, pitchA, offA, afresh, bn, B, ldb, pitchB, bfresh, C, ldc, I, J,
           groups, rpg, alpha, acc, akind="grad", a_n=None):
        """C = alpha * A^T B in the plan's precision (gemm.tn)."""
        return gemm.tn(self.precision, A, lda, A.numel(), B, ldb, B.numel(), C, ldc, I, J, rpg,
                       groups, pitchA, offA, pitchB, alpha, acc, akind,
                       lambda: self.operand(an, A, afresh, akind, a_n),
                       lambda: self.operand(bn, B, bfresh, "act"))

    def tensors(self):
        """Every tensor the plan owns, the GEMM operand buffers included."""
        for v in self.__dict__.values():
            for t in (v if isinstance(v, list) else [v]):
                if isinstance(t, torch.Tensor):
                    yield t
        for op in self._ops.values():
            yield from (t for t in (op.hi, op.lo, op.alpha, op.amax) if t is not None)

    def nbytes(self):
        seen = {t.data_ptr(): t.numel() * t.element_size() for t in self.tensors()}
        return sum(seen.values())


def sinc_constants(k, sr, device):
    """window_ and n_ exactly as SincConv_fast builds them (modules.py:868-876)."""
    n_lin = torch.linspace(0, (k / 2) - 1, steps=int(k / 2))
    window = 0.54 - 0.46 * torch.cos(2 * math.pi * n_lin / k)
    n = (k - 1) / 2.0
    n_ = 2 * math.pi * torch.arange(-n, 0).view(1, -1) / sr
    return n_.reshape(-1).contiguous().to(device), window.contiguous().to(device)


class ParamPack(object):
    """Flat, ordered view of the encoder parameters/buffers handed to the engine."""

    def __init__(self, module):
        self.module = module
        self.names, self.tensors = [], []
        for name, p in module.named_parameters():
            self.names.append(name)
            self.tensors.append(p)
        self.index = {n: i for i, n in enumerate(self.names)}


def _flat(t):
    return t.detach().reshape(-1)


# -- weight preparation shared by encoder_forward and encoder_forward_packed -----------------
def _conv_weight_operands(plan, P):
    """GEMM operands (in the plan's operand format) of every conv block's weight: one launch."""
    jobs = []
    for l, g in enumerate(plan.geoms):
        if not g.sinc:
            hi, lo = plan.w_operand(("Wt", l), plan.Wt[l])
            dst = plan.Wt[l] if plan.precision.fmt == gemm.FMT_F32 else None
            jobs.append((P("blocks.%d.conv.weight" % l), dst, hi, lo, g.Cout, g.Cin, g.k,
                         1, 1, g.Cout * g.Cin * g.k))
    if jobs:
        plan.w_batch(0, jobs)


def _dgrad_weight_operands(plan, P):
    """Data-gradient GEMM operands (in the plan's operand format) of every conv block with an
    input gradient: one launch."""
    jobs = []
    for l, g in enumerate(plan.geoms):
        if not g.sinc and l > 0:
            hi, lo = plan.w_operand(("Wd", l), plan.Wd[l])
            dst = plan.Wd[l] if plan.precision.fmt == gemm.FMT_F32 else None
            jobs.append((P("blocks.%d.conv.weight" % l), dst, hi, lo, g.Cout, g.Cin, g.k,
                         g.s, g.taps, g.s * g.Cin * g.taps * g.Cout))
    if jobs:
        plan.w_batch(1, jobs)


def _sinc_weights(plan, mod, P, l, g, filt=None):
    """The sinc layer's polyphase GEMM operand in plan.Wt[l] (and its band-pass bank in `filt`)
    from low_hz_ / band_hz_."""
    pre = "blocks.%d." % l
    ops.call("pase_sinc_make", P(pre + "conv.low_hz_"), P(pre + "conv.band_hz_"),
             mod._sinc_n, mod._sinc_win, filt, plan.Wt[l], g.Cout, g.k, g.fold, g.K,
             50.0, 50.0, float(plan.cfg["sr"]))


def _sinc_dgrad_weights(plan, mod, P, g):
    """The sinc layer's banded dgrad operand plan.Wdg (DESIGN.md section 17), from the band-pass
    bank regenerated into plan.filt."""
    _sinc_weights(plan, mod, P, g.idx, g, plan.filt)
    ops.call("pase_sinc_dgrad_weight", plan.filt, plan.Wdg, g.Cout, g.k, g.fold, g.dg_rows)


def _sinc_weight_grads(plan, mod, params, g, sink, grads):
    """low_hz_ / band_hz_ gradients from the sinc layer's weight gradient in plan.dWt: written
    into the sink, or new tensors added to `grads`."""
    pre = "blocks.%d." % g.idx
    P = lambda name: _flat(params[name])
    if sink is not None:
        dlow, dband = sink[pre + "conv.low_hz_"], sink[pre + "conv.band_hz_"]
    else:
        dlow = torch.empty_like(params[pre + "conv.low_hz_"])
        dband = torch.empty_like(params[pre + "conv.band_hz_"])
    ops.call("pase_sinc_grad", plan.dWt[g.idx], P(pre + "conv.low_hz_"),
             P(pre + "conv.band_hz_"), mod._sinc_n, mod._sinc_win, dlow.reshape(-1),
             dband.reshape(-1), g.Cout, g.k, g.fold, g.K, 50.0, 50.0, float(plan.cfg["sr"]))
    if sink is None:
        grads[pre + "conv.low_hz_"] = dlow
        grads[pre + "conv.band_hz_"] = dband


def _block_conv_inputs(plan, mod, P, l, g, training):
    """Block l's conv bias (the sinc layer: None, and its band-pass operand regenerated into
    plan.Wt[l]) and, in train mode, its BatchNorm sums in plan.stats_f (else None, None)."""
    if g.sinc:
        _sinc_weights(plan, mod, P, l, g)
        bias = None
    else:
        bias = P("blocks.%d.conv.bias" % l)
    if not training:
        return bias, None, None
    o = plan.fs_off[l]
    return bias, plan.stats_f[o:o + g.Nn], plan.stats_f[o + g.Nn:o + 2 * g.Nn]


def _block_bn(plan, mod, P, l, g, cs, cq, count, counters):
    """Block l's BatchNorm affine into plan.bn[l]: eval mode, from the running statistics, or
    (counters given: train mode) from the sums cs / cq over `count` frames, which also update the
    running statistics; the num_batches_tracked buffer is appended to counters for the caller to
    increment."""
    pre = "blocks.%d." % l
    buf = lambda name: _flat(mod.get_buffer(name))
    mean, invstd, scale, shift = plan.bn[l][0], plan.bn[l][1], plan.bn[l][2], plan.bn[l][3]
    if counters is None:
        ops.call("pase_bn_eval_affine", buf(pre + "norm.running_mean"),
                 buf(pre + "norm.running_var"), P(pre + "norm.weight"), P(pre + "norm.bias"),
                 g.Cout, BN_EPS, mean, invstd, scale, shift)
        return
    ops.call("pase_bn_finalize", cs, cq, g.Cout, g.fold, float(count), P(pre + "norm.weight"),
             P(pre + "norm.bias"), buf(pre + "norm.running_mean"), buf(pre + "norm.running_var"),
             BN_MOMENTUM, BN_EPS, mean, invstd, scale, shift)
    counters.append(mod.get_buffer(pre + "norm.num_batches_tracked"))


def _act_dst(plan, l, xq_row):
    """Where block l's BatchNorm/PReLU pass writes, in the format of the GEMM that reads it:
    (dst, dst_lo, format, row stride, left pad, right pad) of the next block's padded operand, of
    the QRNN input from row xq_row on, or of the output projection's fp32 operand plan.cat."""
    C, fmt = plan.geoms[l].Cout, plan.precision.fmt
    if l + 1 < plan.nblk:
        nx = plan.geoms[l + 1]
        return plan.apad[l + 1], plan.apad_lo[l + 1], fmt, C, nx.padL, nx.padR
    if plan.rnn:
        o = xq_row * C
        return plan.xq[o:], None if plan.xq_lo is None else plan.xq_lo[o:], fmt, C, 0, 0
    return plan.cat, None, gemm.FMT_F32, plan.Kc, 0, 0


def _skip_pool(plan, l, buf):
    """Block l's dense-skip columns of `buf` (the output projection's operand plan.cat or its
    gradient plan.dcat); None for the last block or without dense skips."""
    return buf[plan.col_off[l]:] if plan.skips and l + 1 < plan.nblk else None


def _qrnn_weights(plan, params):
    """Gate weights in the GEMM's [x_{t-1} | x_t] column order."""
    Cq, H = plan.Clast, plan.H
    Wl = params["rnn.layers.0.linear.weight"].detach()
    torch.cat([Wl[:, Cq:], Wl[:, :Cq]], 1, out=plan.Wq.view(3 * H, 2 * Cq))


def _out_weights(plan, params):
    """[W | dense skips] of the output projection."""
    emb = plan.emb
    parts = [params["W.weight"].detach().reshape(emb, -1)]
    if plan.skips:
        parts += [params["denseskips.%d.weight" % i].detach().reshape(emb, -1)
                  for i in range(plan.nblk - 1)]
    torch.cat(parts, 1, out=plan.Wcat.view(emb, plan.Kc))


def _out_bn_eval_affine(plan, buf):
    bo = plan.bn_out
    ops.call("pase_bn_eval_affine", buf("norm_out.running_mean"), buf("norm_out.running_var"),
             None, None, plan.emb, BN_EPS, bo[0], bo[1], bo[2], bo[3])


def _out_proj(plan, mod, params, rows, counters=None):
    """The output projection [W | skips] of the first `rows` frames of plan.cat into plan.yout
    (uniform over the frames) and the norm_out affine into plan.bn_out: eval mode, or (counters
    given: train mode) the statistics of the `rows` frames, whose num_batches_tracked buffer is
    appended to counters for the caller to increment."""
    Kc, emb = plan.Kc, plan.emb
    buf = lambda name: _flat(mod.get_buffer(name))
    _out_weights(plan, params)
    cs = cq = None
    if plan.norm_out and counters is not None:
        o = plan.fs_out
        cs, cq = plan.stats_f[o:o + emb], plan.stats_f[o + emb:o + 2 * emb]
    gemm.nt(plan.precision, plan.cat, Kc, rows * Kc, plan.Wcat, Kc, plan.yout, emb, rows, emb,
            Kc, 1.0, _flat(params["W.bias"]), cs=cs, cq=cq,
            a_op=lambda: plan.operand("cat", plan.cat, True, n=rows * Kc),
            b_op=lambda: plan.operand("Wcat", plan.Wcat, True, "weight"))
    if not plan.norm_out:
        return
    if cs is not None:
        bo = plan.bn_out
        ops.call("pase_bn_finalize", cs, cq, emb, 1, float(rows), None, None,
                 buf("norm_out.running_mean"), buf("norm_out.running_var"), BN_MOMENTUM, BN_EPS,
                 bo[0], bo[1], bo[2], bo[3])
        counters.append(mod.get_buffer("norm_out.num_batches_tracked"))
    else:
        _out_bn_eval_affine(plan, buf)


def encoder_forward(plan, mod, x, params, training, save_for_backward):
    """x: (N,1,T) fp32 CUDA tensor.  params: dict name -> tensor.  Returns
    (out (N,emb,Tq), out_ntc (N*Tq, emb))."""
    call = ops.call
    cfg, G, N = plan.cfg, plan.geoms, plan.N
    Tq, Kc, rows, emb = plan.Tq, plan.Kc, plan.rows, plan.emb
    plan.generation += 1
    P = lambda name: _flat(params[name])
    fmt, ybf = plan.precision.fmt, int(plan.precision.act_bf16)

    g0 = G[0]
    call("pase_reflect_pad_wave", x.reshape(-1), plan.apad[0], plan.apad_lo[0], fmt, N, plan.T,
         g0.padL, g0.padR, g0.apad_floats)
    if training:
        plan.stats_f.zero_()
    if plan.skips:
        plan.cat.zero_()

    _conv_weight_operands(plan, P)
    counters = [] if training else None

    for l, g in enumerate(G):
        bias, cs, cq = _block_conv_inputs(plan, mod, P, l, g, training)
        # sinc: the band-pass operand is regenerated (and converted) every step; conv blocks:
        # pase_conv_w_batch already wrote the operand format
        plan.nt(("apad", l), plan.apad[l], g.lda, False, ("Wt", l), plan.Wt[l], g.K, g.sinc,
                plan.y[l], g.Nn, N * g.P, g.Nn, g.K, 1.0, bias, g.P, g.T_out, g.rows_out,
                g.fold, cs, cq, 0)
        _block_bn(plan, mod, P, l, g, cs, cq, N * g.T_out, counters)
        # the producer writes the next GEMM's operand in its own format (3xTF32: + the tf32
        # residual twin; 3xF16: the fp16 pair); each sample's QRNN input starts at its row 1,
        # row 0 staying zero (its x_{-1})
        C = g.Cout
        dst, dst_lo, dfmt, d_rs, pl, pr = _act_dst(plan, l, 1)
        d_ss = G[l + 1].apad_floats if l + 1 < plan.nblk else (Tq + 1 if plan.rnn else Tq) * d_rs
        pool = _skip_pool(plan, l, plan.cat)
        call("pase_bn_prelu_pad_fwd", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, plan.bn[l][2],
             plan.bn[l][3], P("blocks.%d.act.weight" % l), dst, dst_lo, dfmt, d_ss, d_rs, pl, pr,
             pool, Tq * Kc, Kc, 0 if pool is None else plan.pool_d[l], Tq)

    if plan.rnn:
        Cq, H = plan.Clast, plan.H
        _qrnn_weights(plan, params)
        plan.nt("xq", plan.xq, Cq, False, "Wq", plan.Wq, 2 * Cq, True, plan.Yg, 3 * H,
                N * (Tq + 1), 3 * H, 2 * Cq, 1.0, P("rnn.layers.0.linear.bias"),
                Tq + 1, Tq, Tq, 1, None, None, 0)
        call("pase_qrnn_scan_fwd", plan.Yg, plan.cat, Kc, plan.Cst, N, Tq, H)

    _out_proj(plan, mod, params, rows, counters)
    if counters:                                 # BatchNorm step counters: one launch
        torch._foreach_add_(counters, 1)
    bo = plan.bn_out
    out = torch.empty(N, emb, Tq, dtype=torch.float32, device=x.device)
    out_ntc = torch.empty(rows, emb, dtype=torch.float32, device=x.device)
    call("pase_out_affine_nct", plan.yout, bo[2], bo[3], out.reshape(-1), out_ntc.reshape(-1),
         N, Tq, emb)
    plan.last_training = training
    return out, out_ntc


# -- packed variable-length inference (DESIGN.md section 11) ----------------------------------
INDEX_LIMIT = 2 ** 31          # the packed kernels' tables and row counts are 32-bit ints
MAX_UTTS = 65535               # utterances per pack: the packed kernels give each a grid row
OUT_MODES = {None: 0, "avg_norm": 1, "avg_concat": 2, "avg_norm_concat": 3}


def _accepts(cfg, T):
    try:
        build_geometry(cfg, T)
        return True
    except ValueError:
        return False


def min_length(cfg):
    """Shortest waveform whose every block input is longer than its reflect pads."""
    hi = 1
    while not _accepts(cfg, hi):
        hi *= 2
    lo = hi // 2 + 1 if hi > 1 else 1
    while lo < hi:
        mid = (lo + hi) // 2
        if _accepts(cfg, mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def utterance_geometry(cfg, lengths, sinc_fold):
    """Per-utterance block geometry; an utterance too short for a block's reflect pads raises
    ValueError naming its index (and, from ConvGeom, the block)."""
    out = []
    for i, T in enumerate(lengths):
        try:
            out.append(build_geometry(cfg, T, sinc_fold))
        except ValueError as e:
            raise ValueError("utterance %d (%d samples): %s" % (i, T, e)) from None
    return out


def split_packs(lengths, max_samples, max_count=MAX_UTTS):
    """Greedy, in order: consecutive utterances while their sum fits max_samples and their
    count max_count (at most MAX_UTTS, the packed kernels' grid-row limit); an utterance longer
    than max_samples is a pack of its own.  -> list of (start, stop)."""
    if not 1 <= max_count <= MAX_UTTS:
        raise ValueError("max_count must be in 1..%d, got %r" % (MAX_UTTS, max_count))
    packs, start, total = [], 0, 0
    for i, T in enumerate(lengths):
        if i > start and (total + T > max_samples or i - start >= max_count):
            packs.append((start, i))
            start, total = i, 0
        total += T
    if lengths:
        packs.append((start, len(lengths)))
    return packs


def packed_bounds(geoms, capacity, max_utts):
    """Upper bounds, over every pack of at most `capacity` samples in at most `max_utts`
    utterances, of the elements of each block's padded operand and raw output and of the
    output frames.  Per utterance P = ceil(Tpad / r) <= Tpad / r + 1 and T_out = floor((Tpad -
    k) / s) + 1, so sums over n utterances are bounded through the summed lengths."""
    n = np.arange(1, max_utts + 1, dtype=np.int64)
    L = np.full_like(n, capacity)
    n_apad, n_y = [], []
    for g in geoms:
        r = g.fold if g.sinc else g.s
        Tpad = L + n * (g.padL + g.padR)
        n_apad.append(int(((Tpad // r + n) * g.lda).max()))
        L = (Tpad - n * g.k) // g.s + n
        n_y.append(int(((L // g.fold + n) * g.Nn).max()))
    return n_apad, n_y, int(L.max())


class PackedPlan(EncoderPlan):
    """Forward buffers of packed variable-length inference (encoder_forward_packed) for packs
    of up to `capacity` samples: sized by capacity, not by the lengths in a pack, so one plan
    serves every pack that fits.  Holds the packed waveform and the device copy of the
    per-utterance offset table."""

    def __init__(self, cfg, capacity, device, prec="fp32"):
        self.capacity = int(capacity)
        self.min_len = min_length(cfg)
        self._setup(cfg, device, prec, lambda fold: build_geometry(cfg, self.min_len, fold))
        G = self.geoms
        self.max_utts = min(max(self.capacity // self.min_len, 1), MAX_UTTS)
        n_apad, n_y, rows = packed_bounds(G, self.capacity, self.max_utts)
        sizes = [("waveform", self.capacity)]
        sizes += [("block %d operand" % g.idx, na + g.K + 64) for g, na in zip(G, n_apad)]
        sizes += [("block %d output" % g.idx, ny) for g, ny in zip(G, n_y)]
        sizes += [("output projection operand", rows * self.Kc),
                  ("returned features", 2 * rows * self.emb)]
        if self.rnn:
            sizes += [("QRNN input", (rows + self.max_utts) * self.Clast + 2 * self.Clast + 64),
                      ("QRNN gates", rows * 3 * self.H)]
        _check_indices(self.capacity, sizes)
        self.rows_cap = rows
        self._alloc(n_apad, n_y, rows, rows + self.max_utts)
        self.wave = torch.zeros(self.capacity, dtype=torch.float32, device=device)
        self.table = torch.zeros(_table_size(self.nblk, self.max_utts), dtype=torch.int32,
                                 device=device)


def _check_indices(capacity, sizes):
    """ValueError unless every (what, elements) of a plan for packs of `capacity` samples is
    addressable by the packed kernels' 32-bit indices."""
    for what, n in sizes:
        if n >= INDEX_LIMIT:
            raise ValueError(
                "a pack of %d samples needs %d elements for the %s, beyond the 32-bit indices "
                "of the packed kernels: split it into shorter utterances" % (capacity, n, what))


def _table_size(nblk, n):
    # wave, per block (GEMM map + BN/PReLU rows), QRNN GEMM map, scan, output
    return 3 * n + nblk * (3 * n + 1 + 6 * n) + (3 * n + 1) + 2 * n + 3 * n


def _cum0(a):
    """Exclusive prefix sums over the first axis, with the total as the last row."""
    return np.concatenate([np.zeros((1,) + a.shape[1:], np.int64), np.cumsum(a, 0)])


def _packed_offsets(plan, geoms):
    """Per utterance and block of a pack: rows per sample P and output frames T_out, (n, nblk);
    the first row of every utterance in each block's padded operand (row0) and raw output
    (orow0); its output frames Tq, first output frame q0 and first QRNN input row xr0 (one
    separator row per utterance).  The offsets have n + 1 rows, the last the total."""
    n = len(geoms)
    P = np.array([[g.P for g in gi] for gi in geoms], dtype=np.int64).reshape(n, plan.nblk)
    RO = np.array([[g.rows_out for g in gi] for gi in geoms], dtype=np.int64).reshape(n, -1)
    TO = np.array([[g.T_out for g in gi] for gi in geoms], dtype=np.int64).reshape(n, -1)
    Tq = TO[:, -1]
    return P, TO, _cum0(P), _cum0(RO), Tq, _cum0(Tq), _cum0(Tq + 1)


def packed_layout(plan, lengths, geoms, mode):
    """Offsets of every utterance at every layer, as the int32 table of the packed kernels.
    -> (host table, {section: offset}, dict of sizes).  Utterance i's rows are contiguous at
    every layer; each padded operand starts on a folded-row boundary of its GEMM."""
    G, n = plan.geoms, len(lengths)
    _, TO, row0, orow0, Tq, q0, xr0 = _packed_offsets(plan, geoms)
    E = plan.emb * (2 if mode in ("avg_concat", "avg_norm_concat") else 1)
    o0 = _cum0(E * Tq)
    x0 = _cum0(np.asarray(lengths, dtype=np.int64))
    Kc, sec, parts = plan.Kc, {}, []

    def put(name, *cols, rows=None):
        sec[name] = sum(p.size for p in parts)
        parts.append(np.stack(cols, 1).reshape(-1) if rows is None else np.concatenate(cols))

    put("wave", x0[:n], np.asarray(lengths, np.int64), row0[:n, 0] * G[0].lda)
    for l, g in enumerate(G):
        put(("gemm", l), row0[:, l], orow0[:n, l], TO[:, l], rows=True)
        if l + 1 < plan.nblk:
            dst = row0[:n, l + 1] * G[l + 1].lda
        elif plan.rnn:
            dst = (xr0[:n] + 1) * g.Cout
        else:
            dst = q0[:n] * Kc
        put(("bn", l), TO[:, l], orow0[:n, l] * g.Nn, dst, q0[:n] * Kc,
            np.maximum(TO[:, l] // Tq, 1), Tq)
    put("qgemm", xr0, q0[:n], Tq, rows=True)
    put("scan", q0[:n], Tq)
    put("out", q0[:n], Tq, o0[:n])
    table = np.concatenate(parts)
    assert table.size <= _table_size(plan.nblk, n) and table.max() < INDEX_LIMIT
    sizes = dict(rows=int(q0[n]), xq_rows=int(xr0[n]), gemm_rows=[int(r) for r in row0[n]],
                 max_T=int(max(lengths)), max_Tout=[int(t) for t in TO.max(0)],
                 count=[int(c) for c in TO.sum(0)],
                 out=int(o0[n]), offsets=[int(o) for o in o0[:n]], Tq=[int(t) for t in Tq],
                 E=E)
    return torch.from_numpy(table.astype(np.int32)), sec, sizes


def encoder_forward_packed(plan, mod, x, lengths, geoms, params, mode=None, layout=None,
                           training=False):
    """Forward of utterances packed in x (fp32, sum(lengths) samples, plan.wave).  Eval mode:
    each one computed as a B=1 forward would.  training (DESIGN.md section 19): every BatchNorm
    normalises with the statistics of the valid frames of the whole pack and updates its running
    statistics and counter once.  Launches do not depend on the number of utterances.  Returns
    the list of (1, E, T'_i) features, views of one new buffer.  layout: the table builder
    (default packed_layout; packed_grad_layout also uploads the backward's sections).  Every
    forward bumps plan.generation: a backward saved against an earlier forward of the plan
    raises instead of reading these activations."""
    plan.generation += 1
    counters = [] if training else None
    sz, tab = _packed_front(plan, mod, x, lengths, geoms, params, mode, layout, counters)
    n = len(lengths)
    if plan.rnn:
        ops.call("pase_qrnn_scan_fwd_var", plan.Yg, plan.cat, plan.Kc, plan.Cst, tab("scan"), n,
                 plan.H)
    _out_proj(plan, mod, params, sz["rows"], counters)
    if counters:                                 # BatchNorm step counters: one launch
        torch._foreach_add_(counters, 1)
    bo = plan.bn_out
    out = torch.empty(sz["out"], dtype=torch.float32, device=x.device)
    ops.call("pase_out_affine_var", plan.yout, bo[2], bo[3], out, tab("out"), n, plan.emb,
             OUT_MODES[mode])
    E = sz["E"]
    return [out[o:o + E * t].view(1, E, t) for o, t in zip(sz["offsets"], sz["Tq"])]


def _packed_front(plan, mod, x, lengths, geoms, params, mode, layout=None, counters=None):
    """encoder_forward_packed up to the QRNN scan: every conv block, the pooled skips in
    plan.cat and (rnn configs) the gate pre-activations of every frame in plan.Yg.
    -> (sizes of packed_layout, section -> device table view)."""
    host, sec, sz = (layout or packed_layout)(plan, lengths, geoms, mode)
    plan.table[:host.numel()].copy_(host)                    # the one host-to-device copy
    tab = lambda name: plan.table[sec[name]:]
    _packed_front_launch(plan, mod, x, sz, tab, params, counters)
    return sz, tab


def _packed_front_launch(plan, mod, x, sz, tab, params, counters=None):
    """The launches of _packed_front, from a layout already on the device (tab: section ->
    table view).  counters (a list: train mode): the blocks' BatchNorms use the statistics of
    the pack's sz["count"] valid frames, update their running statistics, and append their
    num_batches_tracked buffers for the caller to increment."""
    training = counters is not None
    call = ops.call
    G, n = plan.geoms, len(sz["Tq"])
    P = lambda name: _flat(params[name])
    fmt, ybf = plan.precision.fmt, int(plan.precision.act_bf16)
    rows, Kc = sz["rows"], plan.Kc

    g0 = G[0]
    call("pase_reflect_pad_wave_var", x, tab("wave"), n, sz["max_T"], plan.apad[0],
         plan.apad_lo[0], fmt, g0.padL, g0.padR)
    if training:
        plan.stats_f.zero_()
    if plan.skips:
        plan.cat[:rows * Kc].zero_()                         # the pools accumulate into it
    _conv_weight_operands(plan, P)
    for l, g in enumerate(G):
        bias, cs, cq = _block_conv_inputs(plan, mod, P, l, g, training)
        plan.nt_var(("apad", l), plan.apad[l], g.lda, ("Wt", l), plan.Wt[l], g.K, g.sinc,
                    plan.y[l], g.Nn, sz["gemm_rows"][l], g.Nn, g.K, bias, tab(("gemm", l)), n,
                    g.fold, cs, cq)
        _block_bn(plan, mod, P, l, g, cs, cq, sz["count"][l], counters)
        # the QRNN input: the table's offsets leave a row ahead of each utterance, which the
        # kernel zeroes (its x_{-1} row)
        dst, dst_lo, dfmt, d_rs, pl, pr = _act_dst(plan, l, 0)
        sep = 1 if plan.rnn and l + 1 == plan.nblk else 0
        call("pase_bn_prelu_pad_fwd_var", plan.y[l], ybf, tab(("bn", l)), n, sz["max_Tout"][l],
             g.Cout, plan.bn[l][2], plan.bn[l][3], P("blocks.%d.act.weight" % l), dst, dst_lo,
             dfmt, d_rs, pl, pr, _skip_pool(plan, l, plan.cat), Kc, sep)

    if plan.rnn:
        Cq, H = plan.Clast, plan.H
        _qrnn_weights(plan, params)
        plan.nt_var("xq", plan.xq, Cq, "Wq", plan.Wq, 2 * Cq, True, plan.Yg, 3 * H,
                    sz["xq_rows"], 3 * H, 2 * Cq, P("rnn.layers.0.linear.bias"), tab("qgemm"), n,
                    1)


# -- packed variable-length backward (DESIGN.md section 18) -----------------------------------
_BWD_ROW = 9            # {T, y_off, a_off, b_off, pool_off, pool_d, pool_T, d_off, d_span}


def _grad_table_size(nblk, n):
    return nblk * _BWD_ROW * n + 3 * n


class PackedGradPlan(PackedPlan):
    """The PackedPlan of WaveFe.encode_packed: the forward buffers of WaveFe.extract, the
    backward's table sections, and backward buffers sized by the capacity bounds, allocated on
    the first differentiated call (the input-gradient ones on the first call returning dx).

    Backward layout: block l's output gradient dyz[l] is the forward operand's row layout
    shifted by `lead` zero rows (taps - 1; sinc: the dgrad halo), so utterance i's frames sit
    at lead + row0[i] and every utterance's zero tail (P_i - T_out_i >= taps - 1 rows) is the
    next one's leading halo.  The dgrad GEMMs then run uniform over sum(P_i) rows into the
    forward operand's layout, and the weight-gradient GEMMs over the same rows as one
    sequence.  The QRNN gate gradient dYg uses the QRNN input's rows: one zero row per
    utterance where the forward reads its separator."""

    def __init__(self, cfg, capacity, device, prec="fp32"):
        super().__init__(cfg, capacity, device, prec)
        G = self.geoms
        n_apad, _, _ = packed_bounds(G, self.capacity, self.max_utts)
        self.n_dxpad = n_apad
        self.grad_rows = [na // g.lda for g, na in zip(G, n_apad)]
        self.yg_rows = self.rows_cap + self.max_utts
        self.n_dyz = [(R + 2 * g.dg_rows) * g.Nn + 128 if g.sinc else
                      (R + 2 * g.taps) * g.Cout + 128 for g, R in zip(G, self.grad_rows)]
        sizes = [("block %d output gradient" % g.idx, nd) for g, nd in zip(G, self.n_dyz)]
        if self.rnn:
            sizes.append(("QRNN gate gradient", self.yg_rows * 3 * self.H + 64))
        _check_indices(self.capacity, sizes)
        self.table = torch.zeros(_table_size(self.nblk, self.max_utts)
                                 + _grad_table_size(self.nblk, self.max_utts),
                                 dtype=torch.int32, device=device)
        self.layout = None            # (sections, sizes) of the last differentiated forward
        self.gflat = self.gzero = None

    def ensure_backward(self):
        if self.backward_ready:
            return
        self._alloc_backward(self.n_dyz, self.n_dxpad, self.rows_cap, self.yg_rows)
        n = self.rows_cap * self.emb
        self.gflat = torch.empty(n, dtype=torch.float32, device=self.device)
        self.gzero = torch.zeros(n, dtype=torch.float32, device=self.device)

    def ensure_input_grad(self):
        self.ensure_backward()
        if self.filt is not None:
            return
        g = self.geoms[0]
        f32 = dict(dtype=torch.float32, device=self.device)
        self.filt = torch.empty(g.Cout * g.k, **f32)
        self.Wdg = torch.empty(g.fold * g.dg_K, **f32)
        self.dxpad[0] = torch.empty(self.grad_rows[0] * g.fold, **f32)


def packed_grad_layout(plan, lengths, geoms, mode=None):
    """packed_layout plus the sections encoder_backward_packed reads: per block ("bwd", l) rows
    of _BWD_ROW ints, and "qbwd" {row0, T, dY row0} of the QRNN scan.  Uploaded with the
    forward's sections in one copy; the plan keeps (sections, sizes) for the backward."""
    host, sec, sz = packed_layout(plan, lengths, geoms, mode)
    G, n = plan.geoms, len(lengths)
    P, TO, row0, orow0, Tq, q0, xr0 = _packed_offsets(plan, geoms)
    Kc, parts, base = plan.Kc, [host.numpy().astype(np.int64)], host.numel()
    zero = np.zeros(n, np.int64)

    def put(name, *cols):
        sec[name] = base + sum(p.size for p in parts[1:])
        parts.append(np.stack(cols, 1).reshape(-1))

    lead = []
    for l, g in enumerate(G):
        C = g.Cout
        if l + 1 < plan.nblk:
            a, b = row0[:n, l + 1] * G[l + 1].lda, zero
        elif plan.rnn:
            a, b = xr0[:n] * 2 * C + C, xr0[:n] * 2 * C
        else:
            a, b = q0[:n] * Kc, zero
        if g.sinc:
            ld = g.dg_halo
            d, span = (ld + g.fold * row0[:n, l]) * C, g.fold * P[:, l]
        else:
            ld = g.taps - 1
            d, span = (ld + row0[:n, l]) * C, P[:, l]
        lead.append(ld)
        put(("bwd", l), TO[:, l], orow0[:n, l] * g.Nn, a, b, q0[:n] * Kc,
            np.maximum(TO[:, l] // Tq, 1), Tq, d, span)
    put("qbwd", q0[:n], Tq, xr0[:n])
    table = np.concatenate(parts)
    assert table.size <= plan.table.numel() and table.max() < INDEX_LIMIT
    sz.update(lead=lead, total=int(sum(lengths)), lengths=[int(T) for T in lengths],
              max_span=[int(m) for m in (np.max(P, 0) * np.array([g.fold for g in G]))])
    plan.layout = (sec, sz)
    return torch.from_numpy(table.astype(np.int32)), sec, sz


def encoder_backward_packed(plan, mod, params, gflat, sink=None, dx=None, param_grads=True,
                            training=False, window=None):
    """Backward of the last packed_grad_layout forward on `plan`, the packed mirror of
    encoder_backward_steps.  gflat: the upstream gradients of the (1, emb, T'_i) outputs,
    concatenated in output order.  dx (optional): the packed (sum T_i,) waveform gradient.
    param_grads / sink / the returned dict as in encoder_backward_steps; the parameter
    gradients are summed over the utterances.  training: the forward used the pack's batch
    statistics, so every BatchNorm's sums S1 / S2 enter the data gradient (DESIGN.md section
    19).  Launches do not depend on the number of utterances.

    window (WaveFe.encode_long, DESIGN.md section 20): the pack is one window of a recording
    recomputed by _window_forward, a dict of _window_backward's.  Then three launches differ:
    the cotangent is the crop's columns of the recording's gradient (gflat unused), the QRNN
    scan carries the cell-state gradient across windows, and dx is the recording's gradient,
    into which the window's waveform gradient is added at its offset."""
    sink, S1o, S2o = _bwd_begin(plan, params, sink, dx, param_grads, "encoder_backward_packed")
    pg = param_grads
    call = ops.call
    sec, sz = plan.layout
    tab = lambda name: plan.table[sec[name]:]
    G, n = plan.geoms, len(sz["Tq"])
    rows, Kc, emb = sz["rows"], plan.Kc, plan.emb
    P = lambda name: _flat(params[name])
    grads, copies = {}, []
    fmt, ybf = plan.precision.fmt, int(plan.precision.act_bf16)
    bo = plan.bn_out
    use_stats = 1 if (plan.norm_out and training) else 0
    if window is not None:
        call("pase_out_bwd_gather_crop", window["gout"], window["ld"], window["col0"], rows,
             window["crop_f0"], window["crop_n"], emb, plan.g)
    elif use_stats:
        call("pase_out_bwd_reduce_var", gflat, tab("out"), n, max(sz["Tq"]), emb, plan.yout,
             bo[0], bo[1], plan.g, S1o, S2o)
    else:
        call("pase_out_bwd_gather_var", gflat, tab("out"), n, max(sz["Tq"]), emb, plan.g)
    _out_bwd(plan, params, sink, copies, grads, pg, S1o, S2o, use_stats, rows, rows * emb)

    if plan.rnn:
        H, R = plan.H, sz["xq_rows"]
        if window is not None:
            call("pase_qrnn_scan_bwd_carry_var", plan.Yg, plan.Cst, plan.dcat, Kc, plan.dYg,
                 window["state"], window["dstate"], tab("qcarry"), 1, H)
        else:
            call("pase_qrnn_scan_bwd_var", plan.Yg, plan.Cst, plan.dcat, Kc, plan.dYg,
                 tab("qbwd"), n, H)
        _qrnn_bwd(plan, sink, copies, grads, pg, R, (R, 0, R, 1, R), R * 3 * H)

    for l in range(plan.nblk - 1, -1, -1):
        g = G[l]
        C, pre, M = g.Cout, "blocks.%d." % l, sz["gemm_rows"][l]
        mean, invstd, scale, shift = plan.bn[l][0], plan.bn[l][1], plan.bn[l][2], plan.bn[l][3]
        # the table's "bwd" rows hold the sample offsets, the QRNN input's x_t columns included
        src = _grad_src(plan, l, ybf, 0) + (_skip_pool(plan, l, plan.dcat), Kc)
        S1, S2, dal, dbi, amax = _bn_grad_sums(plan, l)
        t, mT = tab(("bwd", l)), sz["max_Tout"][l]
        # eval mode: the sums feed parameter gradients only; train mode: the data gradient too
        if pg or amax is not None or training:
            call("pase_bn_prelu_bwd_reduce_var", plan.y[l], ybf, t, n, mT, C, mean, invstd,
                 scale, shift, P(pre + "act.weight"), *src, S1, S2, dal, amax)
        dst = (plan.dyz[l], plan.dyz_lo[l], fmt, sz["lead"][l],
               dbi if pg and not g.sinc else None, amax, plan.gscale[l])
        if training:
            call("pase_bn_prelu_bwd_apply_src_var_train", plan.y[l], ybf, t, n,
                 sz["max_span"][l], C, mean, invstd, P(pre + "norm.weight"), scale, shift,
                 P(pre + "act.weight"), S1, S2, float(sz["count"][l]), *src, *dst)
        else:
            call("pase_bn_prelu_bwd_apply_src_var", plan.y[l], ybf, t, n, sz["max_span"][l], C,
                 invstd, P(pre + "norm.weight"), scale, shift, P(pre + "act.weight"), *src, *dst)
        # one sequence of M rows; dyz[l] leads by sz["lead"][l] frames
        _block_grads(plan, mod, params, sink, grads, pg, l, (M, sz["lead"][l] // g.fold, M, 1, M),
                     (M, M, M, M))
        if g.sinc and dx is not None:
            f = g.fold
            _sinc_dgrad_weights(plan, mod, P, g)
            plan.nt(("dyz", l), plan.dyz[l], g.Nn, False, "Wdg", plan.Wdg, g.dg_K, True,
                    plan.dxpad[0], f, M, f, g.dg_K, 1.0, None, M, M, M, 1, None, None, 0,
                    akind="grad")
            if window is not None:
                call("pase_reflect_fold_wave_acc", plan.dxpad[0], dx, window["seg_start"],
                     sz["total"], g.padL, g.padR, int(window["fold_l"]), int(window["fold_r"]))
            else:
                call("pase_reflect_fold_wave_var", plan.dxpad[0], tab("wave"), n, sz["max_T"],
                     dx, g.padL, g.padR)
    return _bwd_end(plan, sink, copies, grads, pg)


def _bwd_begin(plan, params, sink, dx, param_grads, who):
    """The start of a backward sweep: refuse one with nothing to compute, allocate the backward
    (and, dx given, the input-gradient) buffers, zero the reductions and re-lay out the conv
    weights for the data-gradient GEMMs.  -> (sink, None without parameter gradients; the
    output BatchNorm's sums S1, S2)."""
    if not param_grads and dx is None:
        raise ValueError("%s: nothing to compute (no parameter gradients, no dx)" % who)
    plan.ensure_backward()
    if dx is not None:
        plan.ensure_input_grad()
    sb, o, emb = plan.stats_b, plan.bs_out, plan.emb
    sb.zero_()
    if plan.amax is not None:
        plan.amax.zero_()
    _dgrad_weight_operands(plan, lambda name: _flat(params[name]))
    return sink if param_grads else None, sb[o:o + emb], sb[o + emb:o + 2 * emb]


def _out_bwd(plan, params, sink, copies, grads, pg, S1o, S2o, use_stats, rows, a_n):
    """The output projection's backward from the cotangent of its `rows` frames in plan.g:
    norm_out's backward in place (use_stats: train mode, with the sums S1o / S2o), with
    parameter gradients (pg) the bias sum and the [W | skips] weight gradient, and the gradient
    of plan.cat in plan.dcat.  a_n: elements of plan.g the GEMMs convert (None: all)."""
    call, emb, Kc, bo, sb = ops.call, plan.emb, plan.Kc, plan.bn_out, plan.stats_b
    call("pase_out_bwd_apply", plan.g, plan.yout, bo[0], bo[1], bo[2], S1o, S2o, float(rows),
         use_stats, rows, emb)
    if pg:
        call("pase_colsum", plan.g, emb, rows, emb, sb[plan.bs_bw:plan.bs_bw + emb])
        plan.tn("g", plan.g, emb, rows, 0, True, "cat", plan.cat, Kc, rows, False, plan.dWcat,
                Kc, emb, Kc, 1, rows, 1.0, 0, a_n=a_n)
        _out_weight_grads(plan, plan.geoms, params, sink, copies, grads)
    call("pase_transpose_pad", plan.Wcat, Kc, plan.WcatT, emb, emb, Kc)
    # the weight-gradient GEMM above converted g into the GEMM format; without it, this one does
    plan.nt("g", plan.g, emb, not pg, "WcatT", plan.WcatT, emb, True, plan.dcat, Kc, rows, Kc,
            emb, 1.0, None, rows, rows, rows, 1, None, None, 0, akind="grad", a_n=a_n)


def _qrnn_bwd(plan, sink, copies, grads, pg, M, wmap, a_n):
    """The QRNN's backward after its scan wrote the gate gradients of M rows into plan.dYg: with
    parameter gradients (pg) the bias sum and the gate weight gradient, whose GEMM runs over the
    row map wmap = (pitchA, offA, pitchB, groups, rows_per_group) of dYg and the QRNN input; and
    the gradient of the QRNN input [x_{t-1} | x_t] in plan.dsrc.  a_n as in _out_bwd."""
    Cq, H, sb = plan.Clast, plan.H, plan.stats_b
    if pg:
        pA, oA, pB, groups, rpg = wmap
        ops.call("pase_colsum", plan.dYg, 3 * H, M, 3 * H, sb[plan.bs_bq:plan.bs_bq + 3 * H])
        plan.tn("dYg", plan.dYg, 3 * H, pA, oA, True, "xq", plan.xq, Cq, pB, False, plan.dWq,
                2 * Cq, 3 * H, 2 * Cq, groups, rpg, 1.0, 0, a_n=a_n)
        _qrnn_weight_grads(plan, sink, copies, grads)
    ops.call("pase_transpose_pad", plan.Wq, 2 * Cq, plan.WqT, 3 * H, 3 * H, 2 * Cq)
    plan.nt("dYg", plan.dYg, 3 * H, not pg, "WqT", plan.WqT, 3 * H, True, plan.dsrc, 2 * Cq,
            M, 2 * Cq, 3 * H, 1.0, None, M, M, M, 1, None, None, 0, akind="grad", a_n=a_n)


def _grad_src(plan, l, ybf, x_col):
    """Block l's gradient source (A, A in bf16, A's row stride, left / right pad, B, B's row
    stride, B's row shift): the next block's input gradient plan.dxpad[l + 1] inside its reflect
    pads; for the last block the gradient of the QRNN input (A: its x_t columns from x_col on, B:
    its x_{t-1} columns one row later) or of the output projection's operand, both fp32."""
    if l + 1 < plan.nblk:
        nx = plan.geoms[l + 1]
        return plan.dxpad[l + 1], ybf, plan.geoms[l].Cout, nx.padL, nx.padR, None, 0, 0
    if plan.rnn:
        Cq = plan.Clast
        return plan.dsrc[x_col:], 0, 2 * Cq, 0, 0, plan.dsrc, 2 * Cq, 1
    return plan.dcat, 0, plan.Kc, 0, 0, None, 0, 0


def _bn_grad_sums(plan, l):
    """Block l's reductions in plan.stats_b (S1, S2, dalpha, dbias) and its 3xF16 gradient
    maxima in plan.amax (None in the other precisions)."""
    C, o = plan.geoms[l].Cout, plan.bs_off[l]
    amax = None if plan.amax is None else plan.amax[2 * l:2 * l + 2]
    return (*plan.stats_b[o:o + 4 * C].view(4, C), amax)


def _block_grads(plan, mod, params, sink, grads, pg, l, wmap, dmap):
    """From block l's output gradient in plan.dyz[l]: with parameter gradients (pg) its weight
    gradient (the sinc layer: its cut-off gradients from it), and for conv blocks past the
    first its input gradient in plan.dxpad[l].  wmap = (pitchA, offA, pitchB, groups,
    rows_per_group): the weight-gradient GEMM's row map of dyz[l] and the padded operand; dmap
    = (M, rows_in, t_valid, rows_out): the data-gradient GEMM's."""
    g = plan.geoms[l]
    if pg:
        pA, oA, pB, groups, rpg = wmap
        plan.tn(("dyz", l), plan.dyz[l], g.Nn, pA, oA, False, ("apad", l), plan.apad[l], g.lda,
                pB, False, plan.dWt[l], g.K, g.Nn, g.K, groups, rpg, 1.0, 0)
        if g.sinc:
            _sinc_weight_grads(plan, mod, params, g, sink, grads)
    if not g.sinc and l > 0:
        M, rows_in, t_valid, rows_out = dmap
        C = g.Cout
        plan.nt(("dyz", l), plan.dyz[l], C, False, ("Wd", l), plan.Wd[l], g.taps * C, False,
                plan.dxpad[l], g.s * g.Cin, M, g.s * g.Cin, g.taps * C, 1.0, None, rows_in,
                t_valid, rows_out, 1, None, None, 0, akind="grad")


def _bwd_end(plan, sink, copies, grads, pg):
    """The end of a backward sweep: every parameter gradient written into the sink, or returned
    (autograd); {} when there is none."""
    if not pg:
        return {}
    if sink is not None:
        _emit_sunk_grads(plan, plan.geoms, sink, copies, range(0, plan.nblk), True, "all")
        return {}
    return _autograd_grads(plan, plan.geoms, grads)


def _grad_sink(mod, names):
    """mod.grad_sink (None when unset), refused unless it names every parameter in `names`."""
    sink = getattr(mod, "grad_sink", None)
    if sink is not None and any(nm not in sink for nm in names):
        raise RuntimeError("pase_b200: WaveFe.grad_sink must name every parameter "
                           "(missing %s)" % [nm for nm in names if nm not in sink][:3])
    return sink


def _check_generation(ctx, buffers, later, hint=""):
    """Refuse a backward whose forward's activations in ctx.plan were replaced: every forward
    through a plan bumps its generation, and the forward saved the one it left in ctx."""
    if ctx.plan.generation != ctx.generation:
        raise RuntimeError("pase_b200: %s were overwritten by a later %s before this backward "
                           "ran; run backward before the next forward%s." % (buffers, later, hint))


class _PackedEncoderFn(torch.autograd.Function):
    """Autograd node of WaveFe.encode_packed (eval mode) and WaveFe.encode_packed_train
    (training): one packed forward of n utterances (tensors = the n flat CUDA waveforms, then
    the parameters) and one packed backward sweep.  The outputs are views of one buffer."""

    @staticmethod
    def forward(ctx, mod, plan, lengths, geoms, names, training, n, *tensors):
        params = dict(zip(names, tensors[n:]))
        plan.ensure_backward()
        x = plan.wave[:sum(lengths)]
        torch.cat(tensors[:n], out=x)
        feats = encoder_forward_packed(plan, mod, x, lengths, geoms, params, None,
                                       packed_grad_layout, training)
        ctx.set_materialize_grads(False)
        ctx.mod, ctx.plan, ctx.names, ctx.n, ctx.training = mod, plan, names, n, training
        ctx.generation = plan.generation
        ctx.save_for_backward(*tensors[n:])
        return tuple(feats)

    @staticmethod
    def backward(ctx, *gouts):
        plan, n = ctx.plan, ctx.n
        _check_generation(ctx, "the activation buffers of encode_packed",
                          "encode_packed forward on the same plan")
        params = dict(zip(ctx.names, ctx.saved_tensors))
        need_x = ctx.needs_input_grad[7:7 + n]
        param_grads = any(ctx.needs_input_grad[7 + n:])        # all or nothing, as _EncoderFn
        none = (None,) * 7
        if not param_grads and not any(need_x):
            return none + (None,) * (n + len(ctx.names))
        sink = _grad_sink(ctx.mod, ctx.names)
        sec, sz = plan.layout
        emb = plan.emb
        gflat = plan.gflat[:sz["out"]]
        torch.cat([plan.gzero[:emb * T] if g is None else g.reshape(-1)
                   for g, T in zip(gouts, sz["Tq"])], out=gflat)
        dx = None
        if any(need_x):
            dx = torch.empty(sz["total"], dtype=torch.float32, device=plan.device)
        grads = encoder_backward_packed(plan, ctx.mod, params, gflat, sink, dx, param_grads,
                                        ctx.training)
        dxs, o = [], 0
        for T, need in zip(sz["lengths"], need_x):
            dxs.append(dx[o:o + T] if need else None)
            o += T
        return none + tuple(dxs) + tuple(grads.get(nm) for nm in ctx.names)


# -- windowed inference of one long recording (DESIGN.md section 15) --------------------------
# The whole-recording forward runs the sequential QRNN scan for T' > 512 frames (qrnn.cu
# seg_width); the carried window scan reproduces that one, so a window holds at least 512 frames.
MIN_WINDOW_FRAMES = 512
_TAIL_SEARCH_FRAMES = 2048
_tail_cache = {}


def hop_size(cfg):
    """Samples per output frame: the product of the strides."""
    return int(np.prod(cfg["strides"]))


def min_window(cfg):
    return MIN_WINDOW_FRAMES * hop_size(cfg)


def _block_spans(cfg):
    """Per block (a, b, R): frame t of block l reads samples R*t - a .. R*t + b (R: its stride
    product), composed from the kernels, strides and left reflect pads of ConvGeom."""
    spans, R, a, b = [], 1, 0, 0
    for g in build_geometry(cfg, 1 << 20):
        a, b = R * g.padL + a, R * (g.k - 1 - g.padL) + b
        R *= g.s
        spans.append((a, b, R))
    return spans


def receptive_field(cfg):
    """(A, B): final frame j of a recording depends on samples hop*j - A .. hop*j + B only --
    through the last block and, with dense skips, through the hop/R_l frames of block l pooled
    into it (fuse_skip at its nominal pool factor)."""
    hop, spans = hop_size(cfg), _block_spans(cfg)
    A, B = spans[-1][0], spans[-1][1]
    if cfg["denseskips"]:
        for a, b, R in spans[:-1]:
            A, B = max(A, a), max(B, hop - R + b)
    return A, B


def window_halos(cfg):
    """(left, right) halo in frames: the left one covers A (plus the QRNN's x_{t-1}), the right
    one B beyond the hop of a window's last frame."""
    hop = hop_size(cfg)
    A, B = receptive_field(cfg)
    return _cdiv(A, hop) + (1 if cfg["rnn_pool"] else 0), _cdiv(B + 1 - hop, hop)


def nominal_pool_factors(cfg):
    """fuse_skip's d_l = T_out_l // T' for a long recording: the stride product after block l."""
    s = cfg["strides"]
    return [int(np.prod(s[l + 1:])) for l in range(len(s) - 1)]


def pool_factors(cfg, L):
    G = build_geometry(cfg, L)
    return [max(g.T_out // G[-1].T_out, 1) for g in G[:-1]]


def _tail_table(cfg):
    """(tail, residues): segment lengths L with L mod hop in `residues` never get the nominal
    pool factors (PASE+: L mod 160 >= 151 makes T' = ceil(L/160), so d_0 = 159); in every other
    residue class each length >= tail has them (and valid reflect pads)."""
    key = (tuple(cfg["kwidths"]), tuple(cfg["strides"]), bool(cfg["sincnet"]),
           bool(cfg["denseskips"]))
    if key in _tail_cache:
        return _tail_cache[key]
    hop = hop_size(cfg)
    lens = np.arange(_TAIL_SEARCH_FRAMES * hop, dtype=np.int64)      # row f, column r: f*hop+r
    L, ok, outs = lens, lens > 0, []
    for g in build_geometry(cfg, 1 << 20):
        ok &= (L > g.padL) & (L > g.padR)
        L = (L + g.padL + g.padR - g.k) // g.s + 1
        outs.append(L)
    if cfg["denseskips"]:
        Tq = np.maximum(outs[-1], 1)
        for l, d in enumerate(nominal_pool_factors(cfg)):
            ok &= np.maximum(outs[l] // Tq, 1) == d
    ok = ok.reshape(-1, hop)
    half = ok.shape[0] // 2
    residues = [r for r in range(hop) if not ok[half:, r].all()]
    tail = 1
    for r in range(hop):
        bad = np.nonzero(~ok[:, r])[0]
        if r not in residues and bad.size:
            tail = max(tail, (int(bad[-1]) + 1) * hop + r)
    _tail_cache[key] = (tail, residues)
    return tail, residues


def tail_length(cfg):
    """Shortest segment length from which on every longer one (outside the residues of
    _tail_table) has the nominal pool factors.  A short segment pools skip l over more than d_l
    frames (7597 samples: d_0 = 161 in PASE+), so a recording's last segment is extended to
    this length."""
    return _tail_table(cfg)[0]


def check_windowable(cfg, L):
    """NotImplementedError when a recording of L samples pools its skips at other than the
    nominal factors: its whole-recording frames then drift against any hop-aligned segment."""
    if not cfg["denseskips"]:
        return
    residues = _tail_table(cfg)[1]
    if L % hop_size(cfg) in residues or (L >= tail_length(cfg) and
                                         pool_factors(cfg, L) != nominal_pool_factors(cfg)):
        raise NotImplementedError(
            "a recording of %d samples (%d mod %d) pools its dense skips over %s frames, not the "
            "nominal %s, so no hop-aligned window reproduces its frames; trim or pad it to a "
            "length mod %d outside %d..%d" % (L, L % hop_size(cfg), hop_size(cfg),
                                              pool_factors(cfg, L), nominal_pool_factors(cfg),
                                              hop_size(cfg), min(residues), max(residues)))


def window_capacity(cfg, window):
    """Samples of the longest segment stream_step builds for pieces of stream_chunk(window)
    samples (plan_windows, a StreamPool with that window): window + both halos + one hop + the
    tail extension, whatever the recording's length.  The plan of a FeatureStream and of
    extract_long holds this many samples."""
    hl, hr = window_halos(cfg)
    hop = hop_size(cfg)
    return hop * (window // hop + hl + hr + 1) + tail_length(cfg)


def stream_end(cfg, n):
    """Where a stream's segment ends once n samples have arrived: n, less the last few samples
    when n mod hop falls in the residues without nominal pool factors (_tail_table)."""
    residues, hop = _tail_table(cfg)[1], hop_size(cfg)
    return n - (n % hop - min(residues) + 1) if n % hop in residues else n


def final_frames(cfg, n):
    """Frames of a stream that are final once its first n samples have arrived: frame j reads
    up to sample hop*j + B, and the segment that computes it needs tail_length samples (and a
    length outside the residues of _tail_table: stream_end)."""
    n = stream_end(cfg, n)
    if n < tail_length(cfg):
        return 0
    _, B = receptive_field(cfg)
    return max(0, (n - B - 1) // hop_size(cfg) + 1)


def make_segment(cfg, f0, f1, end):
    """Segment computing frames f0 .. f1-1 from samples up to `end`: starts the left halo before
    f0 on a hop boundary, extended left to tail_length samples (not before 0)."""
    hop, tail = hop_size(cfg), tail_length(cfg)
    s = max(0, f0 - window_halos(cfg)[0]) * hop
    if end - s < tail:
        s = max(0, (end - tail) // hop * hop)
    return dict(seg_start=s, seg_len=end - s, crop_f0=f0 - s // hop, crop_n=f1 - f0)


def check_segment(cfg, seg, at_end):
    """Raise NotImplementedError unless the segment's crop is exactly the whole recording's
    frames (at_end: the segment ends where the recording does)."""
    hop = hop_size(cfg)
    s, n, c0, cn = seg["seg_start"], seg["seg_len"], seg["crop_f0"], seg["crop_n"]
    what = "segment at sample %d (%d samples, frames %d+%d)" % (s, n, c0, cn)
    if s % hop or s < 0 or cn < 1 or c0 < 0:
        raise NotImplementedError("%s: not hop-aligned" % what)
    try:
        G = build_geometry(cfg, n)
    except ValueError as e:
        raise NotImplementedError("%s: %s" % (what, e)) from None
    if c0 + cn > G[-1].T_out:
        raise NotImplementedError("%s: only %d frames" % (what, G[-1].T_out))
    whole = s == 0 and at_end
    if cfg["denseskips"] and not whole and pool_factors(cfg, n) != nominal_pool_factors(cfg):
        raise NotImplementedError("%s: pool factors %s, not the nominal %s"
                                  % (what, pool_factors(cfg, n), nominal_pool_factors(cfg)))
    A, B = receptive_field(cfg)
    lead = 1 if cfg["rnn_pool"] else 0
    if s > 0 and hop * (c0 - lead) - A < 0:
        raise NotImplementedError("%s: left halo short of the receptive field" % what)
    if not at_end and hop * (c0 + cn - 1) + B > n - 1:
        raise NotImplementedError("%s: right halo short of the receptive field" % what)


def stream_step(cfg, n, done, keep, add, at_end=False):
    """The host planner of one stream (FeatureStream, StreamPool), as a pure function of its
    counters: n samples received, frames 0 .. done-1 returned, samples from `keep` on held.
    `add` more samples arrive (at_end: none, and the recording ends at n).  -> (n, done, keep,
    seg) after the step, seg the make_segment dict computing the frames that became final (None
    when none did).  keep is the first sample a later segment can read (its left halo or its
    tail extension).  Raises before anything changes: ValueError for a finish shorter than
    min_length, NotImplementedError for a finish at a length no segment can window or a
    segment that fails check_segment."""
    n += add
    if at_end:
        if n < min_length(cfg):
            raise ValueError("a recording of %d samples is shorter than the encoder's minimum "
                             "of %d" % (n, min_length(cfg)))
        if done > 0:
            check_windowable(cfg, n)
        f1 = frame_counts(cfg, n)[-1]
    else:
        f1 = final_frames(cfg, n)
    if f1 <= done:
        return n, done, keep, None
    seg = make_segment(cfg, done, f1, n if at_end else stream_end(cfg, n))
    check_segment(cfg, seg, at_end)
    hop = hop_size(cfg)
    k = min(max(0, f1 - window_halos(cfg)[0]) * hop,
            max(0, (stream_end(cfg, n) - tail_length(cfg)) // hop * hop))
    return n, f1, max(keep, k), seg


def stream_chunk(cfg, window):
    """Samples of the pieces a stream cuts a longer push into: the window, hop-aligned."""
    return window // hop_size(cfg) * hop_size(cfg)


def stream_ring_capacity(cfg, window):
    """Samples of one stream's history ring in a StreamPool: every sample a segment reads lies
    in keep .. n (at most window_capacity of them, by stream_step) and one call's piece adds at
    most stream_chunk more, so a ring this long never overwrites a sample still to be read."""
    return window_capacity(cfg, window) + stream_chunk(cfg, window)


def plan_windows(cfg, L, window):
    """Segments of a recording of L samples for windows of `window` samples' frames, as
    WaveFe.extract_long runs them: stream_step over pieces of stream_chunk samples, the last one
    at the end of the recording.  A list of dict(seg_start, seg_len, crop_f0, crop_n) whose
    crops tile the recording's frames 0 .. T'-1 once, in order (crop_f0: first frame of the crop
    within the segment).  Host only; raises ValueError for a bad window / a too-short recording
    and NotImplementedError when a segment could not reproduce the whole-recording frames."""
    if window < min_window(cfg):
        raise ValueError("window must be at least %d samples (%d frames), got %d"
                         % (min_window(cfg), MIN_WINDOW_FRAMES, window))
    chunk = stream_chunk(cfg, window)
    pieces = [min(chunk, L - a) for a in range(0, L, chunk)] or [0]
    segs, n, done, keep = [], 0, 0, 0
    for k, add in enumerate(pieces):
        n, done, keep, seg = stream_step(cfg, n, done, keep, add, k + 1 == len(pieces))
        if seg is not None:
            segs.append(seg)
    return segs


# -- gradients through one long recording (DESIGN.md section 20) ----------------------------
def _window_layout(seg):
    """packed_grad_layout of one window (segment `seg`) as a one-utterance pack, plus two
    sections: "carry" {crop_f0, crop_n, 0, 0}, the recomputed scan over the crop from a one-row
    state, and "qcarry" {0, T', 0, crop_f0, crop_n, 0}, its backward."""
    def layout(plan, lengths, geoms, mode=None):
        host, sec, sz = packed_grad_layout(plan, lengths, geoms, mode)
        c0, cn = seg["crop_f0"], seg["crop_n"]
        extra = torch.tensor([c0, cn, 0, 0, 0, sz["Tq"][0], 0, c0, cn, 0], dtype=torch.int32)
        sec["carry"], sec["qcarry"] = host.numel(), host.numel() + 4
        host = torch.cat([host, extra])
        assert host.numel() <= plan.table.numel()
        return host, sec, sz
    return layout


def _window_forward(plan, mod, wav, seg, k, geom, params, log, state):
    """Recompute window k of a recording on `plan` as a one-utterance pack (its samples copied
    into plan.wave): the packed front end, the crop's QRNN scan continued from row k of the
    state log (the sequential body, as the windowed forward ran it) and the output projection.
    Bumps plan.generation, as every forward through a packed plan does."""
    s, n = seg["seg_start"], seg["seg_len"]
    plan.generation += 1
    x = plan.wave[:n]
    x.copy_(wav[s:s + n])
    sz, tab = _packed_front(plan, mod, x, [n], [geom], params, None, _window_layout(seg))
    if plan.rnn:
        if not plan.skips:        # frames outside the crop: no scan writes their QRNN columns
            plan.cat[:sz["rows"] * plan.Kc].zero_()
        state.copy_(log[k])
        ops.call("pase_qrnn_scan_fwd_carry_var", plan.Yg, plan.cat, plan.Kc, plan.Cst, state,
                 tab("carry"), 1, plan.H)
    _out_proj(plan, mod, params, sz["rows"])


def _window_backward(plan, mod, params, wav, segs, log, gout, dx, param_grads, sink):
    """Backward of a recording windowed into `segs` (plan_windows) whose forward logged the
    QRNN state entering each window in `log` (nseg, H): the windows in reverse order, each
    recomputed (_window_forward) and differentiated by encoder_backward_packed with a cotangent
    that is zero outside its crop.  The cell-state gradient is carried from each window to the
    one before it; dx (the recording's, zeroed) accumulates every window's waveform gradient.
    param_grads: the gradients of every parameter are summed over the windows in fp32, in a
    fixed order (last window first), into one flat buffer; then they go to `sink` (a dict of destinations, written
    once) or are returned as a dict of views of that buffer."""
    cfg, H, emb = plan.cfg, plan.H, plan.emb
    hop, L = hop_size(cfg), wav.numel()
    geoms = utterance_geometry(cfg, [sg["seg_len"] for sg in segs], plan.precision.sinc_fold)
    T = gout.shape[-1]
    gout = gout.reshape(emb, T).contiguous()
    f32 = dict(dtype=torch.float32, device=plan.device)
    state = torch.empty(max(H, 1), **f32)
    dstate = torch.zeros(max(H, 1), **f32)
    acc = part = None
    if param_grads:
        names = list(params)
        sizes = [params[nm].numel() for nm in names]
        acc, part = torch.empty(sum(sizes), **f32), torch.empty(sum(sizes), **f32)
        views = lambda flat: dict(zip(names, [v.view(params[nm].shape) for nm, v in
                                              zip(names, flat.split(sizes))]))
        acc_sink, part_sink = views(acc), views(part)
    for k in range(len(segs) - 1, -1, -1):
        seg = segs[k]
        _window_forward(plan, mod, wav, seg, k, geoms[k], params, log, state)
        s, n = seg["seg_start"], seg["seg_len"]
        win = dict(gout=gout, ld=T, col0=s // hop + seg["crop_f0"], crop_f0=seg["crop_f0"],
                   crop_n=seg["crop_n"], state=log[k], dstate=dstate, seg_start=s, fold_l=s == 0,
                   fold_r=s + n == L)
        first = k == len(segs) - 1
        encoder_backward_packed(plan, mod, params, None,
                                (acc_sink if first else part_sink) if param_grads else None,
                                dx, param_grads, window=win)
        if param_grads and not first:
            ops.call("pase_axpy", part, acc, acc.numel(), 1.0)
    if not param_grads:
        return {}
    if sink is None:
        return acc_sink
    rows = [[acc_sink[nm].data_ptr(), sink[nm].data_ptr(), 1, acc_sink[nm].numel(),
             acc_sink[nm].numel(), acc_sink[nm].numel()] for nm in acc_sink]
    table = torch.tensor(rows, dtype=torch.int64).reshape(-1).to(plan.device)
    ops.call("pase_scatter_copy", table, len(rows), acc.numel())
    return {}


class _LongEncoderFn(torch.autograd.Function):
    """Autograd node of WaveFe.encode_long: the windowed forward of one recording (a one-stream
    StreamPool push, as WaveFe.extract_long runs it) with the QRNN state entering each window
    logged, and a backward that recomputes the windows one at a time (_window_backward).
    Saves the waveform, the parameters, the state log and the host window list; no
    activation."""

    @staticmethod
    def forward(ctx, mod, pool, window, segs, names, x, *tensors):
        L, H, emb = x.numel(), pool.plan.H, mod.emb_dim
        T = frame_counts(mod.cfg, L)[-1]
        out = torch.empty(emb, T, dtype=torch.float32, device=x.device)
        log = torch.zeros(len(segs), max(H, 1), dtype=torch.float32, device=x.device)
        sid = pool.open()
        try:
            pool._push({sid: x}, [sid], out, iter(log))
        finally:
            pool._release(sid)
        ctx.set_materialize_grads(False)
        ctx.mod, ctx.window, ctx.segs, ctx.names, ctx.log = mod, window, segs, names, log
        ctx.save_for_backward(x, *tensors)
        return out.view(1, emb, T)

    @staticmethod
    def backward(ctx, gout):
        x, *tensors = ctx.saved_tensors        # raises if any was modified in place since
        need_x = ctx.needs_input_grad[5]
        param_grads = any(ctx.needs_input_grad[6:])          # all or nothing, as _EncoderFn
        none = (None,) * 5
        if gout is None or not (need_x or param_grads):
            return none + (None,) * (1 + len(tensors))
        mod = ctx.mod
        sink = _grad_sink(mod, ctx.names) if param_grads else None
        plan = mod._grad_plan(window_capacity(mod.cfg, ctx.window), x.device)
        mod._sinc_consts(x.device)
        dx = torch.zeros(x.numel(), dtype=torch.float32, device=x.device) if need_x else None
        params = dict(zip(ctx.names, tensors))
        grads = _window_backward(plan, mod, params, x, ctx.segs, ctx.log, gout, dx, param_grads,
                                 sink)
        return none + (dx,) + tuple(grads.get(nm) for nm in ctx.names)


def encoder_backward(plan, mod, params, gout, gntc, training, sink=None, dx=None,
                     param_grads=True):
    """Returns dict name -> gradient tensor (fp32, parameter shape); see
    encoder_backward_steps (this runs it to completion)."""
    gen = encoder_backward_steps(plan, mod, params, gout, gntc, training, sink, dx=dx,
                                 param_grads=param_grads)
    try:
        while True:
            next(gen)
    except StopIteration as done:
        return done.value


def encoder_backward_steps(plan, mod, params, gout, gntc, training, sink=None, split=None,
                           dx=None, param_grads=True):
    """Generator form of the backward sweep.  Returns (StopIteration.value) dict name ->
    gradient tensor (fp32, parameter shape).

    dx (optional): (N,1,T) fp32 tensor that receives the gradient of the input waveform
    (_sinc_input_grad).  param_grads=False (a frozen encoder, dx given) runs the data-gradient
    sweep only: no weight-gradient GEMM, pase_sinc_grad, bias colsum, weight re-layout, cast or
    sink write; it returns {}.  The BatchNorm/PReLU reductions stay: in train mode their sums
    enter the data gradient.

    split (sink mode only): block index s.  The generator yields ONCE, after every gradient
    of the output layer, the QRNN and blocks >= s has been written to its sink destination
    (their re-layout / cast / scatter launches are issued before the yield) and before the
    backward of blocks s-1 .. 0 is launched.  Data parallelism starts the all-reduce of that
    (large) part of the flat gradient buffer on a side stream at the yield and hides it behind
    the remaining backward, which contains the two largest activations (pase_b200/graph.py).

    sink (optional): dict name -> destination tensor (fp32, parameter shape, contiguous, e.g.
    views of the flat gradient buffer of pase_b200.optim.FlatAdam).  When given for every
    parameter, the gradients are WRITTEN (not accumulated) there by the kernels themselves --
    conv weight gradients by the batched re-layout, the sinc cut-offs by pase_sinc_grad,
    everything else by one batched strided copy -- and {} is returned: no per-parameter
    clones, no autograd accumulation kernels, no packing before the all-reduce."""
    sink, S1o, S2o = _bwd_begin(plan, params, sink, dx, param_grads, "encoder_backward_steps")
    pg = param_grads
    call = ops.call
    G, N = plan.geoms, plan.N
    Tq, Kc, rows, emb = plan.Tq, plan.Kc, plan.rows, plan.emb
    P = lambda name: _flat(params[name])
    grads = {}
    copies = []          # sink mode: (src tensor view, rows, cols, src_ld, destination name)
    fmt, ybf = plan.precision.fmt, int(plan.precision.act_bf16)
    zeros = plan.zeros64
    bo = plan.bn_out
    call("pase_out_bwd_reduce", None if gout is None else gout.reshape(-1),
         None if gntc is None else gntc.reshape(-1), plan.yout, bo[0], bo[1], N, Tq, emb,
         plan.g, S1o, S2o)
    use_stats = 1 if (plan.norm_out and training) else 0
    _out_bwd(plan, params, sink, copies, grads, pg, S1o, S2o, use_stats, rows, None)

    if plan.rnn:
        call("pase_qrnn_scan_bwd", plan.Yg, plan.Cst, plan.dcat, Kc, plan.dYg, N, Tq, plan.H)
        # the weight-gradient GEMM: N samples of Tq gate rows against Tq + 1 input rows
        _qrnn_bwd(plan, sink, copies, grads, pg, rows, (Tq, 0, Tq + 1, N, Tq), None)

    if split is not None and (sink is None or not (0 < split < plan.nblk)):
        raise ValueError("encoder_backward_steps: split needs sink mode and 0 < split < nblk")
    for l in range(plan.nblk - 1, -1, -1):
        if split is not None and l == split - 1:
            # everything above is final: emit the upper part of the gradients, then hand control
            # back (the caller launches the collective of that bucket)
            _emit_sunk_grads(plan, G, sink, copies, range(split, plan.nblk), True, "hi")
            copies = []
            yield "upper"
        g = G[l]
        C = g.Cout
        pre = "blocks.%d." % l
        mean, invstd, scale, shift = plan.bn[l][0], plan.bn[l][1], plan.bn[l][2], plan.bn[l][3]
        # per sample: the last block's sources (dsrc / dcat) hold Tq rows
        A, a_bf16, a_rs, padL, padR, B, b_rs, b_shift = _grad_src(plan, l, ybf, plan.Clast)
        a_ss = G[l + 1].apad_floats if l + 1 < plan.nblk else Tq * a_rs
        pool = _skip_pool(plan, l, plan.dcat)
        pd = 0 if pool is None else plan.pool_d[l]
        # dyz[l] per sample: `pitch` rows, the first `lead` of them zero
        lead, pitch = (0, g.rows_out) if g.sinc else (g.taps - 1, g.Pd)
        d_ss = pitch * g.Nn
        dst = plan.dyz[l][lead * C:]
        dst_lo = None if plan.dyz_lo[l] is None else plan.dyz_lo[l][lead * C:]
        S1, S2, dal, dbi, amax = _bn_grad_sums(plan, l)
        # pass 1 writes only its sums; pass 2 recomputes du = PReLU'(u) g from the same
        # gradient sources (no du tensor: one activation-sized write + read less per block)
        src = (A, a_bf16, a_ss, a_rs, padL, padR, B, Tq * b_rs, b_rs, b_shift, pool, Tq * Kc, Kc,
               pd, Tq)
        call("pase_bn_prelu_bwd_reduce", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, mean, invstd,
             scale, shift, P(pre + "act.weight"), *src, None, d_ss, S1, S2, dal, amax)
        if training:
            a1, a2 = S1, S2
        else:
            a1, a2 = zeros[:C], zeros[C:2 * C]
        call("pase_bn_prelu_bwd_apply_src", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, mean, invstd,
             P(pre + "norm.weight"), scale, shift, P(pre + "act.weight"), a1, a2,
             float(N * g.T_out), *src, dst, dst_lo, fmt, d_ss, None if g.sinc else dbi, amax,
             plan.gscale[l])
        _block_grads(plan, mod, params, sink, grads, pg, l, (pitch, lead, g.P, N, g.rows_out),
                     (N * g.Pd, g.Pd, g.P, g.P))
        if g.sinc and dx is not None:
            _sinc_input_grad(plan, mod, P, g, dx)

    if split is not None:
        _emit_sunk_grads(plan, G, sink, copies, range(0, split), False, "lo")
        return {}
    return _bwd_end(plan, sink, copies, grads, pg)


def _out_weight_grads(plan, G, params, sink, copies, grads):
    """[W | skips] weight gradient in plan.dWcat -> sink copies or autograd gradients."""
    emb, Kc = plan.emb, plan.Kc
    dWcat = plan.dWcat.view(emb, Kc)
    first = plan.H if plan.rnn else plan.Clast
    if sink is not None:
        copies.append((dWcat, emb, first, Kc, "W.weight"))
        if plan.skips:
            for i in range(plan.nblk - 1):
                copies.append((dWcat[:, plan.col_off[i]:], emb, G[i].Cout, Kc,
                               "denseskips.%d.weight" % i))
    else:
        # gradients handed to autograd must not alias plan-owned buffers (the next backward
        # would overwrite them): copy the slices out
        grads["W.weight"] = dWcat[:, :first].clone().reshape(params["W.weight"].shape)
        if plan.skips:
            for i in range(plan.nblk - 1):
                c0 = plan.col_off[i]
                grads["denseskips.%d.weight" % i] = \
                    dWcat[:, c0:c0 + G[i].Cout].clone().reshape(
                        params["denseskips.%d.weight" % i].shape)


def _qrnn_weight_grads(plan, sink, copies, grads):
    """QRNN gate weight gradient in plan.dWq -> sink copies or an autograd gradient."""
    Cq, H = plan.Clast, plan.H
    dWq = plan.dWq.view(3 * H, 2 * Cq)
    if sink is not None:          # [x_{t-1} | x_t] GEMM order -> the parameter's [x_t | x_{t-1}]
        dst = sink["rnn.layers.0.linear.weight"].view(3 * H, 2 * Cq)
        copies.append((dWq[:, Cq:], 3 * H, Cq, 2 * Cq, dst))
        copies.append((dWq, 3 * H, Cq, 2 * Cq, dst[:, Cq:]))
    else:
        grads["rnn.layers.0.linear.weight"] = torch.cat([dWq[:, Cq:], dWq[:, :Cq]], 1)


def _autograd_grads(plan, G, grads):
    """Autograd mode, after the sweep: the conv weight and small gradients added to `grads`."""
    call = ops.call
    sb = plan.stats_b
    # conv weight gradients: GEMM layout -> parameter layout for every block in one launch,
    # into one per-call buffer (the gradients handed to autograd are views of it)
    conv_blocks = [l for l, g in enumerate(G) if not g.sinc]
    jobs, off = [], 0
    for l in conv_blocks:
        g = G[l]
        cnt = g.Cout * g.Cin * g.k
        jobs.append((plan.dWt[l], off, None, None, g.Cout, g.Cin, g.k, 1, 1, cnt))
        off += cnt
    if jobs:
        dWflat = torch.empty(off, dtype=torch.float32, device=plan.device)
        plan.w_batch(2, jobs, dWflat)
        for (_, o, _, _, Cout, Cin, k, _, _, cnt), l in zip(jobs, conv_blocks):
            grads["blocks.%d.conv.weight" % l] = dWflat[o:o + cnt].view(Cout, Cin, k)
    # one cast for every small reduction (double accumulators -> fp32 gradients) into a
    # per-call vector; the per-parameter gradients are views of it (no copies)
    gv = torch.empty_like(plan.grad_vec)
    call("pase_cast_d2f", sb, gv, sb.numel(), 1.0)
    grads.update(_small_grad_views(plan, G, gv, range(plan.nblk), True))
    return grads


def _sinc_input_grad(plan, mod, P, g, dx):
    """dx (N,1,T) fp32 = the waveform gradient, from the sinc layer's output gradient in
    plan.dyz[0] (DESIGN.md section 17): the band-pass bank regenerated from low_hz_ / band_hz_,
    its banded dgrad operand, a copy of dy with a zero halo around every sample, one polyphase
    GEMM into the padded-waveform gradient and the reflect fold-back."""
    call, N, f, p = ops.call, plan.N, g.fold, plan.precision
    _sinc_dgrad_weights(plan, mod, P, g)
    call("pase_sinc_dgrad_pack", plan.dyz[0], plan.dyz_lo[0], plan.dyh, plan.dyh_lo, p.esz, N,
         g.Cout, g.T_out, g.Ty, g.dg_halo, g.dg_P * f)
    plan.nt(("dyh", 0), plan.dyh, g.Nn, False, "Wdg", plan.Wdg, g.dg_K, True, plan.dxpad[0], f,
            N * g.dg_P, f, g.dg_K, 1.0, None, g.dg_P, g.P, g.P, 1, None, None, 0, akind="grad")
    call("pase_reflect_fold_wave", plan.dxpad[0], g.P * f, dx.reshape(-1), N, plan.T, g.padL,
         g.padR)


def _small_grad_views(plan, G, gv, layers, top):
    """Views into the cast reduction vector: BatchNorm / PReLU / bias gradients of `layers`
    (+ the output-side biases when `top`)."""
    small = {}
    for l in layers:
        g = G[l]
        C, o = g.Cout, plan.bs_off[l]
        pre = "blocks.%d." % l
        small[pre + "norm.bias"] = gv[o:o + C]
        small[pre + "norm.weight"] = gv[o + C:o + 2 * C]
        small[pre + "act.weight"] = gv[o + 2 * C:o + 3 * C]
        if not g.sinc:
            small[pre + "conv.bias"] = gv[o + 3 * C:o + 4 * C]
    if top:
        small["W.bias"] = gv[plan.bs_bw:plan.bs_bw + plan.emb]
        if plan.rnn:
            small["rnn.layers.0.linear.bias"] = gv[plan.bs_bq:plan.bs_bq + 3 * plan.H]
    return small


def _emit_sunk_grads(plan, G, sink, copies, layers, top, tag):
    """Sink mode: write the gradients of `layers` (+ output-side tensors when `top`) into their
    destinations: conv weights by the batched re-layout (offsets relative to the lowest sink
    address), everything else by ONE batched strided copy."""
    call = ops.call
    base = min(sink.values(), key=lambda t: t.data_ptr())
    base_ptr = base.data_ptr()
    jobs = []
    for l in layers:
        g = G[l]
        if g.sinc:
            continue
        d = sink["blocks.%d.conv.weight" % l]
        jobs.append((plan.dWt[l], (d.data_ptr() - base_ptr) // 4, None, None, g.Cout, g.Cin, g.k,
                     1, 1, g.Cout * g.Cin * g.k))
    if jobs:
        plan.w_batch(2, jobs, base, key=("from_fwd", tag))
    gv = plan.grad_vec
    sb = plan.stats_b
    call("pase_cast_d2f", sb, gv, sb.numel(), 1.0)
    copies = list(copies)
    for name, t in _small_grad_views(plan, G, gv, layers, top).items():
        copies.append((t, 1, t.numel(), t.numel(), name))
    rows = []
    for (src, r, c, sld, dst) in copies:
        d = sink[dst] if isinstance(dst, str) else dst
        dld = c if isinstance(dst, str) else d.stride(0)
        rows.append([src.data_ptr(), d.data_ptr(), r, c, sld, dld])
    ent = plan._wtables.get(("scatter", tag))
    if ent is None or ent[0] != rows:
        ent = (rows, torch.tensor(rows, dtype=torch.int64).reshape(-1).to(plan.device))
        plan._wtables[("scatter", tag)] = ent
    call("pase_scatter_copy", ent[1], len(rows), sum(r[2] * r[3] for r in rows))


class _EncoderFn(torch.autograd.Function):
    """Whole-encoder autograd node: one forward / one backward sweep over the
    plan's buffers (no per-op autograd graph)."""

    @staticmethod
    def forward(ctx, x, mod, plan, training, names, *tensors):
        params = dict(zip(names, tensors))
        plan.ensure_backward()
        out, out_ntc = encoder_forward(plan, mod, x, params, training, True)
        ctx.mod, ctx.plan, ctx.training, ctx.names = mod, plan, training, names
        ctx.generation = plan.generation
        ctx.save_for_backward(*tensors)
        return out, out_ntc

    @staticmethod
    def backward(ctx, gout, gntc):
        plan = ctx.plan
        _check_generation(ctx, "the encoder's activation buffers",
                          "forward of the same (N,T) shape", " (or build a second WaveFe instance)")
        params = dict(zip(ctx.names, ctx.saved_tensors))
        if gout is not None:
            gout = gout.contiguous()
        if gntc is not None:
            gntc = gntc.contiguous()
        sink = _grad_sink(ctx.mod, ctx.names)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(plan.N, 1, plan.T, dtype=torch.float32, device=plan.device)
        # all or nothing: one parameter that needs a gradient runs the full sweep
        param_grads = any(ctx.needs_input_grad[5:])
        grads = encoder_backward(plan, ctx.mod, params, gout, gntc, ctx.training, sink, dx=dx,
                                 param_grads=param_grads)
        return (dx, None, None, None, None) + tuple(grads.get(n) for n in ctx.names)
