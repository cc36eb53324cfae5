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
import os
import torch

from . import ops

BN_EPS = 1e-5
BN_MOMENTUM = 0.1
SINC_FOLD = 4            # polyphase fold of the sinc layer on the fp32 FFMA path
# on the tensor-core path one folded row = one 128-byte TMA row: 32 fp32 / 64 16-bit elements
TC_SINC_FOLD = {0: 32, 1: 32, 2: 64, 3: 64}
# numerics of the GEMMs (pase_tc_gemm_* `mode`): None = fp32 FFMA; 0 = TF32; 1 = 3xTF32
# (fp32-equivalent); 2 = bf16 operands AND bf16 activation storage; 3 = 3xF16 (fp16 operand
# pairs, fp32-equivalent products at half the tensor time / operand bytes of 3xTF32)
PRECISIONS = {"fp32": None, "3xtf32": 1, "tf32": 0, "bf16": 2, "3xf16": 3}
# storage format codes of the C-ABI (include/pase_b200.h)
FMT_F32, FMT_BF16, FMT_F16X2 = 0, 1, 2
OP_FMT = {None: FMT_F32, 0: FMT_F32, 1: FMT_F32, 2: FMT_BF16, 3: FMT_F16X2}
OP_DTYPE = {None: torch.float32, 0: torch.float32, 1: torch.float32, 2: torch.bfloat16,
            3: torch.float16}


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


class Operand(object):
    """One GEMM operand in the format of the plan's GEMM mode.
    hi / lo: the tensors handed to pase_tc_gemm_* (lo None outside the split modes);
    alpha: device float[2] = {1/s, s} when the operand is a power-of-two scaled gradient
    (3xF16), else None;  src: the fp32 tensor it is converted from (None when the producing
    kernel writes the operand format directly)."""
    __slots__ = ("hi", "lo", "alpha", "src", "kind", "amax")

    def __init__(self, hi, lo=None, alpha=None, src=None, kind="act", amax=None):
        self.hi, self.lo, self.alpha, self.src, self.kind, self.amax = hi, lo, alpha, src, kind, amax


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
        self.cfg, self.N, self.T, self.device = cfg, N, T, device
        if prec not in PRECISIONS:
            raise ValueError("precision must be one of %s" % (sorted(PRECISIONS),))
        self.prec, self.mode = prec, PRECISIONS[prec]
        mode = self.mode
        self.fmt = OP_FMT[mode]
        self.op_dtype = OP_DTYPE[mode]
        self.split_mode = mode in (1, 3)
        self.y_bf16 = 1 if mode == 2 else 0
        self.eb = 64 if mode in (2, 3) else 32          # elements per 128-byte TMA row
        self._ops = {}
        self._wtables = {}
        self.geoms = build_geometry(cfg, T, TC_SINC_FOLD[mode] if mode is not None else SINC_FOLD)
        G = self.geoms
        if mode in (2, 3):
            for g in G:
                if (g.lda % 64) or (g.Cout % 64 and not g.sinc):
                    raise NotImplementedError(
                        "precision %r needs channel counts that are multiples of 64 (block %d: "
                        "Cin=%d Cout=%d stride=%d)" % (prec, g.idx, g.Cin, g.Cout, g.s))
        self.nblk = len(G)
        self.Tq = G[-1].T_out
        self.emb = cfg["emb_dim"]
        self.rnn = bool(cfg["rnn_pool"])
        self.skips = bool(cfg["denseskips"])
        self.norm_out = bool(cfg["norm_out"])
        self.Clast = G[-1].Cout
        self.H = (cfg["rnn_dim"] // 2) * 2 if self.rnn else 0
        f32 = dict(dtype=torch.float32, device=device)
        f64 = dict(dtype=torch.float64, device=device)
        opd = dict(dtype=self.op_dtype, device=device)
        yd = dict(dtype=torch.bfloat16 if mode == 2 else torch.float32, device=device)
        z = lambda n: torch.zeros(int(n), **f32)
        e = lambda n: torch.empty(int(n), **f32)
        zo = lambda n: torch.zeros(int(n), **opd)          # operand-format buffers (hi / lo)
        zlo = lambda n: torch.zeros(int(n), **opd) if self.split_mode else None

        # concatenated [rnn-out | pooled skips] operand of the output projection
        self.col_off = []
        off = self.H if self.rnn else self.Clast
        for g in G[:-1]:
            self.col_off.append(off)
            if self.skips:
                off += g.Cout
        self.Kc = off
        self.pool_d = [max(g.T_out // self.Tq, 1) for g in G[:-1]]

        self.apad, self.apad_lo, self.y, self.bn = [], [], [], []
        self.Wt = []
        for g in G:
            n_apad = N * g.apad_floats + g.K + 64
            self.apad.append(zo(n_apad))
            self.apad_lo.append(zlo(n_apad))
            self._ops[("apad", g.idx)] = Operand(self.apad[-1], self.apad_lo[-1])
            self.y.append(torch.empty(int(N * g.rows_out * g.Nn), **yd))
            self.bn.append(torch.zeros(4, g.Cout, **f32))       # mean, invstd, scale, shift
            self.Wt.append(e(g.Nn * g.K))
        rows = N * self.Tq
        self.rows = rows
        if self.rnn:
            Cq, H = self.Clast, self.H
            n_xq = N * (self.Tq + 1) * Cq + 2 * Cq + 64
            self.xq, self.xq_lo = zo(n_xq), zlo(n_xq)
            self._ops["xq"] = Operand(self.xq, self.xq_lo)
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
        self.generation = 0

    def ensure_backward(self):
        """Allocate the backward-only buffers (input / output gradients in operand format,
        weight-gradient and dgrad-weight layouts, fp64 reduction accumulators).  Called by
        WaveFe.encode before a forward that will be differentiated, i.e. during the eager
        warm-up steps and never inside a CUDA-graph capture."""
        if self.backward_ready:
            return
        G, N, mode, device = self.geoms, self.N, self.mode, self.device
        f32 = dict(dtype=torch.float32, device=device)
        f64 = dict(dtype=torch.float64, device=device)
        opd = dict(dtype=self.op_dtype, device=device)
        yd = dict(dtype=torch.bfloat16 if mode == 2 else torch.float32, device=device)
        z = lambda n: torch.zeros(int(n), **f32)
        e = lambda n: torch.empty(int(n), **f32)
        zo = lambda n: torch.zeros(int(n), **opd)
        zlo = lambda n: torch.zeros(int(n), **opd) if self.split_mode else None
        self.dWt, self.Wd, self.dyz, self.dyz_lo, self.dxpad, self.gscale = [], [], [], [], [], []
        for g in G:
            self.dWt.append(e(g.Nn * g.K))
            gs = torch.ones(2, **f32) if mode == 3 else None
            self.gscale.append(gs)
            if g.sinc:
                n_dyz = N * g.rows_out * g.Nn + 128
                self.Wd.append(None)
                self.dxpad.append(None)
            else:
                n_dyz = N * g.Pd * g.Cout + g.taps * g.Cout + 128
                self.Wd.append(e(g.s * g.Cin * g.taps * g.Cout))
                self.dxpad.append(torch.empty(int(N * g.apad_floats), **yd) if g.idx > 0 else None)
            self.dyz.append(zo(n_dyz))
            self.dyz_lo.append(zlo(n_dyz))
            self._ops[("dyz", g.idx)] = Operand(self.dyz[-1], self.dyz_lo[-1],
                                                None if gs is None else gs, kind="grad")
        rows = self.rows
        if self.rnn:
            Cq, H = self.Clast, self.H
            self.dYg = z(rows * 3 * H + 64)
            self.dsrc = e(rows * 2 * Cq)
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
        self.amax = torch.zeros(2 * (self.nblk + 4), **f32) if mode == 3 else None
        self.backward_ready = True

    # -- GEMM operands -----------------------------------------------------------------
    def operand(self, name, buf, fresh=True, kind="act"):
        """Operand `name` in the plan's GEMM format.  Operands whose producer writes the GEMM
        format directly (apad, xq, dyz) are registered at construction; everything else is an
        fp32 tensor converted here (`fresh=False` reuses this step's earlier conversion):
          tf32   : the tensor itself;
          3xtf32 : activations: the tensor is "hi" (tf32 tensor cores truncate), lo = rn(x-trunc(x));
                   weights: explicit hi = rn(x), lo = rn(x - hi) (no coherent bias);
          bf16   : bf16 copy;    3xf16 : fp16 (hi, lo') pair, gradients pre-scaled by a power
                   of two (alpha = {1/s, s} on the device)."""
        op = self._ops.get(name)
        if op is not None and op.src is None:
            return op
        mode = self.mode
        if mode == 0:
            return Operand(buf)
        if op is None or op.src.numel() != buf.numel() or op.src.data_ptr() != buf.data_ptr():
            f32 = dict(dtype=torch.float32, device=self.device)
            if mode == 1:
                hi = torch.zeros_like(buf) if kind == "weight" else buf
                op = Operand(hi, torch.zeros_like(buf), src=buf, kind=kind)
            elif mode == 2:
                op = Operand(torch.zeros(buf.numel(), dtype=torch.bfloat16, device=self.device),
                             src=buf, kind=kind)
            else:
                h = torch.zeros(buf.numel(), dtype=torch.float16, device=self.device)
                grad = kind == "grad"
                op = Operand(h, torch.zeros_like(h),
                             torch.ones(2, **f32) if grad else None, src=buf, kind=kind,
                             amax=torch.zeros(2, **f32) if grad else None)
            self._ops[name] = op
            fresh = True
        if fresh:
            n = buf.numel()
            if mode == 1:
                ops.call("pase_split_tf32", buf, op.hi if kind == "weight" else None, op.lo, n)
            elif mode == 2:
                ops.call("pase_cast_bf16", buf, op.hi, n)
            else:
                if op.amax is not None:
                    op.amax.zero_()
                    ops.call("pase_absmax", buf, n, op.amax)
                ops.call("pase_split_f16", buf, op.hi, op.lo, n, op.amax, op.alpha)
        return op

    def w_operand(self, name, buf):
        """(hi, lo) buffers of a weight operand written by pase_conv_w_batch itself."""
        mode = self.mode
        if mode is None or mode == 0:
            return None, None
        op = self._ops.get(name)
        if op is None:
            if mode == 1:
                op = Operand(torch.zeros_like(buf), torch.zeros_like(buf))
            elif mode == 2:
                op = Operand(torch.zeros(buf.numel(), dtype=torch.bfloat16, device=self.device))
            else:
                h = torch.zeros(buf.numel(), dtype=torch.float16, device=self.device)
                op = Operand(h, torch.zeros_like(h))
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
        fmt = {1: 0, 2: 1, 3: 2}.get(self.mode, 0)
        if tiled:
            ops.call("pase_conv_w_batch", ent[1], len(rows), blocks, op + 3, dst_base, fmt)
        else:
            ops.call("pase_conv_w_batch", ent[1], len(rows), start, op, dst_base, fmt)

    def _tc_ok(self, *elem_strides):
        """Tensor-core path: every operand row stride must be a multiple of 16 bytes (and the
        A operand's folded row a multiple of 128 bytes -- checked by the caller)."""
        q = 8 if self.mode in (2, 3) else 4
        return all(s % q == 0 for s in elem_strides)

    def nt(self, an, A, lda, afresh, bn, B, ldb, bfresh, C, ldc, M, N, K, alpha, bias,
           rows_in, t_valid, rows_out, fold, cs, cq, acc, akind="act"):
        """C = alpha * A B^T (+ bias): tensor-core kernel in the plan's GEMM mode, or the fp32
        FFMA kernel (precision fp32, or shapes the TMA path cannot address)."""
        direct = an in self._ops and self._ops[an].src is None      # no fp32 copy exists
        if self.mode is None or lda % self.eb != 0 or not self._tc_ok(K, ldb):
            if direct and self.mode in (2, 3):
                raise NotImplementedError("precision %r: GEMM shape (lda=%d K=%d) outside the "
                                          "tensor-core path" % (self.prec, lda, K))
            return ops.call("pase_gemm_nt", A, lda, B, ldb, C, ldc, M, N, K, alpha, bias,
                            rows_in, t_valid, rows_out, fold, cs, cq, acc)
        a = self.operand(an, A, afresh, akind)
        b = self.operand(bn, B, bfresh, "weight")
        c16 = 1 if C.dtype == torch.bfloat16 else 0
        return ops.call("pase_tc_gemm_nt", a.hi, a.lo, a.hi.numel() // lda, lda, b.hi, b.lo, ldb,
                        C, ldc, M, N, K, alpha, None if a.alpha is None else a.alpha, bias,
                        rows_in, t_valid, rows_out, fold, cs, cq, acc, self.mode, c16)

    def tn(self, an, A, lda, pitchA, offA, afresh, bn, B, ldb, pitchB, bfresh, C, ldc, I, J,
           groups, rpg, alpha, acc, akind="grad"):
        direct = (an in self._ops and self._ops[an].src is None) or \
            (bn in self._ops and self._ops[bn].src is None)
        if self.mode is None or ldb % self.eb != 0 or not self._tc_ok(lda) or I % 4 != 0 or \
                J % self.eb != 0:
            if direct and self.mode in (2, 3):
                raise NotImplementedError("precision %r: weight-gradient GEMM shape (lda=%d "
                                          "ldb=%d I=%d J=%d) outside the tensor-core path"
                                          % (self.prec, lda, ldb, I, J))
            return ops.call("pase_gemm_tn", A, lda, pitchA, offA, B, ldb, pitchB, 0, C, ldc, I, J,
                            groups, rpg, alpha, acc)
        a = self.operand(an, A, afresh, akind)
        b = self.operand(bn, B, bfresh, "act")
        return ops.call("pase_tc_gemm_tn", a.hi, a.lo, lda, pitchA, offA, b.hi, b.lo, ldb, pitchB,
                        b.hi.numel() // ldb, C, ldc, I, J, groups, rpg, alpha,
                        None if a.alpha is None else a.alpha, acc, self.mode)

    def nbytes(self):
        tot, seen = 0, set()

        def add(t):
            nonlocal tot
            if isinstance(t, torch.Tensor) and t.data_ptr() not in seen:
                seen.add(t.data_ptr())
                tot += t.numel() * t.element_size()
        for v in self.__dict__.values():
            for t in (v if isinstance(v, list) else [v]):
                add(t)
        for op in self._ops.values():
            add(op.hi)
            add(op.lo)
        return tot


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


def encoder_forward(plan, mod, x, params, training, save_for_backward):
    """x: (N,1,T) fp32 CUDA tensor.  params: dict name -> tensor.  Returns
    (out (N,emb,Tq), out_ntc (N*Tq, emb))."""
    call = ops.call
    cfg, G, N = plan.cfg, plan.geoms, plan.N
    Tq, Kc, rows, emb = plan.Tq, plan.Kc, plan.rows, plan.emb
    plan.generation += 1
    P = lambda name: _flat(params[name])
    buf = lambda name: _flat(mod.get_buffer(name))
    fmt, ybf = plan.fmt, plan.y_bf16

    g0 = G[0]
    call("pase_reflect_pad_wave", x.reshape(-1), plan.apad[0], plan.apad_lo[0], fmt, N, plan.T,
         g0.padL, g0.padR, g0.apad_floats)
    if training:
        plan.stats_f.zero_()
    if plan.skips:
        plan.cat.zero_()

    # GEMM operands (in the plan's operand format) of every conv block's weight: one launch
    jobs = []
    for l, g in enumerate(G):
        if not g.sinc:
            hi, lo = plan.w_operand(("Wt", l), plan.Wt[l])
            dst = plan.Wt[l] if plan.mode in (None, 0, 1) else None
            jobs.append((P("blocks.%d.conv.weight" % l), dst, hi, lo, g.Cout, g.Cin, g.k,
                         1, 1, g.Cout * g.Cin * g.k))
    if jobs:
        plan.w_batch(0, jobs)
    counters = []

    for l, g in enumerate(G):
        pre = "blocks.%d." % l
        if g.sinc:
            call("pase_sinc_make", P(pre + "conv.low_hz_"), P(pre + "conv.band_hz_"),
                 mod._sinc_n, mod._sinc_win, None, plan.Wt[l], g.Cout, g.k, g.fold, g.K,
                 50.0, 50.0, float(cfg["sr"]))
            bias = None
        else:
            bias = P(pre + "conv.bias")
        if training:
            o = plan.fs_off[l]
            cs, cq = plan.stats_f[o:o + g.Nn], plan.stats_f[o + g.Nn:o + 2 * g.Nn]
        else:
            cs = cq = None
        # sinc: the band-pass operand is regenerated (and converted) every step; conv blocks:
        # pase_conv_w_batch already wrote the operand format
        plan.nt(("apad", l), plan.apad[l], g.lda, False, ("Wt", l), plan.Wt[l], g.K, g.sinc,
                plan.y[l], g.Nn, N * g.P, g.Nn, g.K, 1.0, bias, g.P, g.T_out, g.rows_out,
                g.fold, cs, cq, 0)
        mean, invstd, scale, shift = plan.bn[l][0], plan.bn[l][1], plan.bn[l][2], plan.bn[l][3]
        if training:
            call("pase_bn_finalize", cs, cq, g.Cout, g.fold, float(N * g.T_out),
                 P(pre + "norm.weight"), P(pre + "norm.bias"),
                 buf(pre + "norm.running_mean"), buf(pre + "norm.running_var"),
                 BN_MOMENTUM, BN_EPS, mean, invstd, scale, shift)
            counters.append(mod.get_buffer(pre + "norm.num_batches_tracked"))
        else:
            call("pase_bn_eval_affine", buf(pre + "norm.running_mean"),
                 buf(pre + "norm.running_var"), P(pre + "norm.weight"), P(pre + "norm.bias"),
                 g.Cout, BN_EPS, mean, invstd, scale, shift)
        C = g.Cout
        # the producer writes the next GEMM's operand in its own format (3xTF32: + the tf32
        # residual twin; 3xF16: the fp16 pair)
        if l + 1 < plan.nblk:
            nx = G[l + 1]
            dst, dst_lo, dfmt = plan.apad[l + 1], plan.apad_lo[l + 1], fmt
            d_ss, d_rs, pl, pr = nx.apad_floats, C, nx.padL, nx.padR
        elif plan.rnn:
            dst, dfmt = plan.xq[C:], fmt
            dst_lo = None if plan.xq_lo is None else plan.xq_lo[C:]
            d_ss, d_rs, pl, pr = (Tq + 1) * C, C, 0, 0
        else:
            dst, dst_lo, dfmt, d_ss, d_rs, pl, pr = plan.cat, None, FMT_F32, Tq * Kc, Kc, 0, 0
        if plan.skips and l + 1 < plan.nblk:
            pool, pd = plan.cat[plan.col_off[l]:], plan.pool_d[l]
        else:
            pool, pd = None, 0
        call("pase_bn_prelu_pad_fwd", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, scale, shift,
             P(pre + "act.weight"), dst, dst_lo, dfmt, d_ss, d_rs, pl, pr, pool, Tq * Kc, Kc, pd,
             Tq)

    if plan.rnn:
        Cq, H = plan.Clast, plan.H
        Wl = params["rnn.layers.0.linear.weight"].detach()
        Wq = plan.Wq.view(3 * H, 2 * Cq)
        torch.cat([Wl[:, Cq:], Wl[:, :Cq]], 1, out=Wq)               # [x_{t-1} | x_t] order
        plan.nt("xq", plan.xq, Cq, False, "Wq", plan.Wq, 2 * Cq, True, plan.Yg, 3 * H,
                N * (Tq + 1), 3 * H, 2 * Cq, 1.0, P("rnn.layers.0.linear.bias"),
                Tq + 1, Tq, Tq, 1, None, None, 0)
        call("pase_qrnn_scan_fwd", plan.Yg, plan.cat, Kc, plan.Cst, N, Tq, H)

    parts = [params["W.weight"].detach().reshape(emb, -1)]
    if plan.skips:
        parts += [params["denseskips.%d.weight" % i].detach().reshape(emb, -1)
                  for i in range(plan.nblk - 1)]
    torch.cat(parts, 1, out=plan.Wcat.view(emb, Kc))
    use_stats = plan.norm_out and training
    if use_stats:
        o = plan.fs_out
        cs, cq = plan.stats_f[o:o + emb], plan.stats_f[o + emb:o + 2 * emb]
    else:
        cs = cq = None
    plan.nt("cat", plan.cat, Kc, True, "Wcat", plan.Wcat, Kc, True, plan.yout, emb,
            rows, emb, Kc, 1.0, P("W.bias"), rows, rows, rows, 1, cs, cq, 0)
    bo = plan.bn_out
    if plan.norm_out:
        if training:
            call("pase_bn_finalize", cs, cq, emb, 1, float(rows), None, None,
                 buf("norm_out.running_mean"), buf("norm_out.running_var"),
                 BN_MOMENTUM, BN_EPS, bo[0], bo[1], bo[2], bo[3])
            counters.append(mod.get_buffer("norm_out.num_batches_tracked"))
        else:
            call("pase_bn_eval_affine", buf("norm_out.running_mean"),
                 buf("norm_out.running_var"), None, None, emb, BN_EPS,
                 bo[0], bo[1], bo[2], bo[3])
    if counters:                                 # BatchNorm step counters: one launch
        torch._foreach_add_(counters, 1)
    out = torch.empty(N, emb, Tq, dtype=torch.float32, device=x.device)
    out_ntc = torch.empty(rows, emb, dtype=torch.float32, device=x.device)
    call("pase_out_affine_nct", plan.yout, bo[2], bo[3], out.reshape(-1), out_ntc.reshape(-1),
         N, Tq, emb)
    plan.last_training = training
    return out, out_ntc


def encoder_backward(plan, mod, params, gout, gntc, training, sink=None):
    """Returns dict name -> gradient tensor (fp32, parameter shape); see
    encoder_backward_steps (this runs it to completion)."""
    gen = encoder_backward_steps(plan, mod, params, gout, gntc, training, sink)
    try:
        while True:
            next(gen)
    except StopIteration as done:
        return done.value


def encoder_backward_steps(plan, mod, params, gout, gntc, training, sink=None, split=None):
    """Generator form of the backward sweep.  Returns (StopIteration.value) dict name ->
    gradient tensor (fp32, parameter shape).

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
    plan.ensure_backward()
    call = ops.call
    cfg, G, N = plan.cfg, plan.geoms, plan.N
    Tq, Kc, rows, emb = plan.Tq, plan.Kc, plan.rows, plan.emb
    P = lambda name: _flat(params[name])
    grads = {}
    sb = plan.stats_b
    sb.zero_()
    if plan.amax is not None:
        plan.amax.zero_()
    fmt, ybf = plan.fmt, plan.y_bf16
    # dgrad operands (operand format) of every conv block with an input gradient: one launch
    jobs = []
    for l, g in enumerate(G):
        if not g.sinc and l > 0:
            hi, lo = plan.w_operand(("Wd", l), plan.Wd[l])
            dst = plan.Wd[l] if plan.mode in (None, 0, 1) else None
            jobs.append((P("blocks.%d.conv.weight" % l), dst, hi, lo, g.Cout, g.Cin, g.k,
                         g.s, g.taps, g.s * g.Cin * g.taps * g.Cout))
    if jobs:
        plan.w_batch(1, jobs)
    zeros = plan.zeros64
    bo = plan.bn_out
    o = plan.bs_out
    S1o, S2o = sb[o:o + emb], sb[o + emb:o + 2 * emb]
    call("pase_out_bwd_reduce", None if gout is None else gout.reshape(-1),
         None if gntc is None else gntc.reshape(-1), plan.yout, bo[0], bo[1], N, Tq, emb,
         plan.g, S1o, S2o)
    use_stats = 1 if (plan.norm_out and training) else 0
    call("pase_out_bwd_apply", plan.g, plan.yout, bo[0], bo[1], bo[2], S1o, S2o, float(rows),
         use_stats, rows, emb)
    call("pase_colsum", plan.g, emb, rows, emb, sb[plan.bs_bw:plan.bs_bw + emb])
    plan.tn("g", plan.g, emb, rows, 0, True, "cat", plan.cat, Kc, rows, False, plan.dWcat, Kc,
            emb, Kc, 1, rows, 1.0, 0)
    call("pase_transpose_pad", plan.Wcat, Kc, plan.WcatT, emb, emb, Kc)
    plan.nt("g", plan.g, emb, False, "WcatT", plan.WcatT, emb, True, plan.dcat, Kc, rows, Kc,
            emb, 1.0, None, rows, rows, rows, 1, None, None, 0, akind="grad")
    dWcat = plan.dWcat.view(emb, Kc)
    first = plan.H if plan.rnn else plan.Clast
    copies = []          # sink mode: (src tensor view, rows, cols, src_ld, destination name)
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

    Cl = plan.Clast
    if plan.rnn:
        Cq, H = Cl, plan.H
        call("pase_qrnn_scan_bwd", plan.Yg, plan.Cst, plan.dcat, Kc, plan.dYg, N, Tq, H)
        call("pase_colsum", plan.dYg, 3 * H, rows, 3 * H, sb[plan.bs_bq:plan.bs_bq + 3 * H])
        plan.tn("dYg", plan.dYg, 3 * H, Tq, 0, True, "xq", plan.xq, Cq, Tq + 1, False,
                plan.dWq, 2 * Cq, 3 * H, 2 * Cq, N, Tq, 1.0, 0)
        dWq = plan.dWq.view(3 * H, 2 * Cq)
        if sink is not None:        # [x_{t-1} | x_t] GEMM order -> the parameter's [x_t | x_{t-1}]
            dst = sink["rnn.layers.0.linear.weight"].view(3 * H, 2 * Cq)
            copies.append((dWq[:, Cq:], 3 * H, Cq, 2 * Cq, dst))
            copies.append((dWq, 3 * H, Cq, 2 * Cq, dst[:, Cq:]))
        else:
            grads["rnn.layers.0.linear.weight"] = torch.cat([dWq[:, Cq:], dWq[:, :Cq]], 1)
        call("pase_transpose_pad", plan.Wq, 2 * Cq, plan.WqT, 3 * H, 3 * H, 2 * Cq)
        plan.nt("dYg", plan.dYg, 3 * H, False, "WqT", plan.WqT, 3 * H, True, plan.dsrc, 2 * Cq,
                rows, 2 * Cq, 3 * H, 1.0, None, rows, rows, rows, 1, None, None, 0, akind="grad")
        last_src = dict(A=plan.dsrc[Cq:], a_ss=Tq * 2 * Cq, a_rs=2 * Cq,
                        B=plan.dsrc, b_ss=Tq * 2 * Cq, b_rs=2 * Cq, b_shift=1)
    else:
        last_src = dict(A=plan.dcat, a_ss=Tq * Kc, a_rs=Kc, B=None, b_ss=0, b_rs=0, b_shift=0)

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
        if l == plan.nblk - 1:
            s = dict(last_src)
            s.update(padL=0, padR=0, a_bf16=0)          # dsrc / dcat are fp32 in every mode
        else:
            nx = G[l + 1]
            s = dict(A=plan.dxpad[l + 1], a_ss=nx.apad_floats, a_rs=C, padL=nx.padL,
                     padR=nx.padR, B=None, b_ss=0, b_rs=0, b_shift=0, a_bf16=ybf)
        if plan.skips and l + 1 < plan.nblk:
            pool, pd = plan.dcat[plan.col_off[l]:], plan.pool_d[l]
        else:
            pool, pd = None, 0
        doff = 0 if g.sinc else (g.taps - 1) * C
        d_ss = g.Ty * C if g.sinc else g.Pd * C
        dst = plan.dyz[l][doff:]
        dst_lo = None if plan.dyz_lo[l] is None else plan.dyz_lo[l][doff:]
        amax = None if plan.amax is None else plan.amax[2 * l:2 * l + 2]
        o = plan.bs_off[l]
        S1, S2, dal, dbi = sb[o:o + C], sb[o + C:o + 2 * C], sb[o + 2 * C:o + 3 * C], \
            sb[o + 3 * C:o + 4 * C]
        # pass 1 writes only its sums; pass 2 recomputes du = PReLU'(u) g from the same
        # gradient sources (no du tensor: one activation-sized write + read less per block)
        src = (s["A"], s["a_bf16"], s["a_ss"], s["a_rs"], s["padL"], s["padR"],
               s["B"], s["b_ss"], s["b_rs"], s["b_shift"], pool, Tq * Kc, Kc, pd, Tq)
        if os.environ.get("PASE_B200_BN_DU") == "1":      # debug: two passes with a stored du
            du = torch.empty(N * d_ss + 64, dtype=plan.y[l].dtype, device=plan.y[l].device)
            call("pase_bn_prelu_bwd_reduce", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, mean, invstd,
                 scale, shift, P(pre + "act.weight"), *src, du, d_ss, S1, S2, dal, amax)
            call("pase_bn_prelu_bwd_apply", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, mean, invstd,
                 P(pre + "norm.weight"), S1 if training else zeros[:C],
                 S2 if training else zeros[C:2 * C], float(N * g.T_out), du, dst, dst_lo, fmt, d_ss,
                 None if g.sinc else dbi, amax, plan.gscale[l])
            _bn_du_debug = True
        else:
            _bn_du_debug = False
            call("pase_bn_prelu_bwd_reduce", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, mean, invstd,
                 scale, shift, P(pre + "act.weight"), *src, None, d_ss, S1, S2, dal, amax)
        if training:
            a1, a2 = S1, S2
        else:
            a1, a2 = zeros[:C], zeros[C:2 * C]
        if not _bn_du_debug:
          call("pase_bn_prelu_bwd_apply_src", plan.y[l], ybf, g.Ty * C, N, g.T_out, C, mean, invstd,
             P(pre + "norm.weight"), scale, shift, P(pre + "act.weight"), a1, a2,
             float(N * g.T_out), *src, dst, dst_lo, fmt, d_ss, None if g.sinc else dbi, amax,
             plan.gscale[l])
        if g.sinc:
            plan.tn(("dyz", l), plan.dyz[l], g.Nn, g.rows_out, 0, False, ("apad", l), plan.apad[l],
                    g.lda, g.P, False, plan.dWt[l], g.K, g.Nn, g.K, N, g.rows_out, 1.0, 0)
            if sink is not None:
                dlow, dband = sink[pre + "conv.low_hz_"], sink[pre + "conv.band_hz_"]
            else:
                dlow = torch.empty_like(params[pre + "conv.low_hz_"])
                dband = torch.empty_like(params[pre + "conv.band_hz_"])
            call("pase_sinc_grad", plan.dWt[l], P(pre + "conv.low_hz_"),
                 P(pre + "conv.band_hz_"), mod._sinc_n, mod._sinc_win, dlow.reshape(-1),
                 dband.reshape(-1), g.Cout, g.k, g.fold, g.K, 50.0, 50.0, float(cfg["sr"]))
            if sink is None:
                grads[pre + "conv.low_hz_"] = dlow
                grads[pre + "conv.band_hz_"] = dband
        else:
            plan.tn(("dyz", l), plan.dyz[l], C, g.Pd, g.taps - 1, False, ("apad", l), plan.apad[l],
                    g.lda, g.P, False, plan.dWt[l], g.K, C, g.K, N, g.T_out, 1.0, 0)
            if l > 0:
                plan.nt(("dyz", l), plan.dyz[l], C, False, ("Wd", l), plan.Wd[l], g.taps * C, False,
                        plan.dxpad[l], g.s * g.Cin, N * g.Pd, g.s * g.Cin, g.taps * C, 1.0, None,
                        g.Pd, g.P, g.P, 1, None, None, 0, akind="grad")

    if sink is not None:
        if split is not None:
            _emit_sunk_grads(plan, G, sink, copies, range(0, split), False, "lo")
        else:
            _emit_sunk_grads(plan, G, sink, copies, range(0, plan.nblk), True, "all")
        return {}

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
        if plan.generation != ctx.generation:
            raise RuntimeError(
                "pase_b200: the encoder's activation buffers were overwritten by a later "
                "forward of the same (N,T) shape before this backward ran; run backward "
                "before the next forward (or build a second WaveFe instance).")
        params = dict(zip(ctx.names, ctx.saved_tensors))
        if gout is not None:
            gout = gout.contiguous()
        if gntc is not None:
            gntc = gntc.contiguous()
        sink = getattr(ctx.mod, "grad_sink", None)
        if sink is not None and any(n not in sink for n in ctx.names):
            raise RuntimeError("pase_b200: WaveFe.grad_sink must name every parameter "
                               "(missing %s)" % [n for n in ctx.names if n not in sink][:3])
        grads = encoder_backward(plan, ctx.mod, params, gout, gntc, ctx.training, sink)
        return (None, None, None, None, None) + tuple(grads.get(n) for n in ctx.names)
