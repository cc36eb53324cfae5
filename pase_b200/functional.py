"""Differentiable building blocks of the worker heads over the C-ABI kernels.

Tensors are channel-last "row" matrices (rows = sample*time, columns =
channels) with a leading dimension that is a multiple of 4 floats; padding
columns are kept at zero so a padded matrix can be fed straight back as a GEMM
operand.  Each autograd Function launches only kernels of pase_b200/csrc.
"""
import os

import torch

from . import ops

# GEMM numerics of the heads (same meaning as WaveFe.precision): "3xf16" / "3xtf32" (wgmma,
# fp32-equivalent products), "tf32", "bf16" (bf16 operands, fp32 everything else), or "fp32"
# (FFMA kernels).
PRECISION = os.environ.get("PASE_B200_PRECISION", "3xf16")
_MODES = {"fp32": None, "3xtf32": 1, "tf32": 0, "bf16": 2, "3xf16": 3}


def set_precision(p):
    global PRECISION
    if p not in _MODES:
        raise ValueError("precision must be one of %s" % sorted(_MODES))
    PRECISION = p


def _ru4(n):
    return (n + 3) // 4 * 4


def _ru(n, m):
    return (n + m - 1) // m * m


def _eb(mode):
    """elements per 128-byte TMA row of the GEMM operands"""
    return 64 if mode in (2, 3) else 32


def _pad_ld(n):
    """leading dimension of a rows-matrix with n columns: tensor-core modes pad to one
    128-byte row so the matrix can itself be a TMA operand."""
    mode = _MODES[PRECISION]
    return _ru4(n) if mode is None else _ru(n, _eb(mode))


class Operand(object):
    """A GEMM operand converted to the current mode's format: hi / lo tensors + the device
    scalar that undoes a gradient's power-of-two scale (3xF16)."""
    __slots__ = ("hi", "lo", "alpha")

    def __init__(self, hi, lo=None, alpha=None):
        self.hi, self.lo, self.alpha = hi, lo, alpha


def to_operand(flat, n, mode, kind="act"):
    """flat: fp32 1-D view (>= n elements).  kind: 'act' | 'weight' | 'grad'."""
    if isinstance(flat, Operand):
        return flat
    dev = flat.device
    if mode == 0:
        return Operand(flat)
    if mode == 1:
        lo = torch.empty(n, dtype=torch.float32, device=dev)
        if kind == "weight":
            hi = torch.empty(n, dtype=torch.float32, device=dev)
            ops.call("pase_split_tf32", flat, hi, lo, n)
            return Operand(hi, lo)
        ops.call("pase_split_tf32", flat, None, lo, n)
        return Operand(flat, lo)
    if mode == 2:
        hi = torch.empty(n, dtype=torch.bfloat16, device=dev)
        ops.call("pase_cast_bf16", flat, hi, n)
        return Operand(hi)
    hi = torch.empty(n, dtype=torch.float16, device=dev)
    lo = torch.empty(n, dtype=torch.float16, device=dev)
    if kind == "grad":
        amax = torch.zeros(2, dtype=torch.float32, device=dev)
        scale = torch.empty(2, dtype=torch.float32, device=dev)
        ops.call("pase_absmax", flat, n, amax)
        ops.call("pase_split_f16", flat, hi, lo, n, amax, scale)
        return Operand(hi, lo, scale)
    ops.call("pase_split_f16", flat, hi, lo, n, None, None)
    return Operand(hi, lo)


def gemm_nt(A, lda, a_used, B, ldb, b_used, C, ldc, M, N, K, bias, rows_in=None, t_valid=None,
            rows_out=None, a_kind="act"):
    """C[map(m),n] = sum_k A[m*lda+k] B[n*ldb+k] + bias[n]; dispatches wgmma / FFMA.
    Optional row map (rows_in, t_valid, rows_out) as in pase_gemm_nt.  A / B may be fp32 flat
    views or already-converted Operands."""
    mode = _MODES[PRECISION]
    if rows_in is None:
        rows_in = t_valid = rows_out = M
    esz = 2 if mode in (2, 3) else 4
    if mode is None or lda % _eb(mode) != 0 or (K * esz) % 16 != 0 or (ldb * esz) % 16 != 0:
        assert not isinstance(A, Operand) and not isinstance(B, Operand)
        return ops.call("pase_gemm_nt", A, lda, B, ldb, C, ldc, M, N, K, 1.0, bias,
                        rows_in, t_valid, rows_out, 1, None, None, 0)
    a = to_operand(A, a_used, mode, a_kind)
    b = to_operand(B, b_used, mode, "weight")
    return ops.call("pase_tc_gemm_nt", a.hi, a.lo, a_used // lda, lda, b.hi, b.lo, ldb, C, ldc,
                    M, N, K, 1.0, a.alpha, bias, rows_in, t_valid, rows_out, 1, None, None, 0,
                    mode, 0)


def gemm_tn(A, lda, a_used, B, ldb, b_used, C, ldc, I, J, rows, groups=1, pitchA=None, offA=0,
            pitchB=None, a_kind="grad"):
    """C[i,j] = sum_r A[rowA(r)*lda+i] B[rowB(r)*ldb+j] over `groups` x `rows` rows."""
    mode = _MODES[PRECISION]
    pitchA = rows if pitchA is None else pitchA
    pitchB = rows if pitchB is None else pitchB
    esz = 2 if mode in (2, 3) else 4
    if mode is None or ldb % _eb(mode) != 0 or (lda * esz) % 16 != 0 or I % 4 != 0 or \
            J % _eb(mode) != 0:
        assert not isinstance(A, Operand) and not isinstance(B, Operand)
        return ops.call("pase_gemm_tn", A, lda, pitchA, offA, B, ldb, pitchB, 0, C, ldc, I, J,
                        groups, rows, 1.0, 0)
    a = to_operand(A, a_used, mode, a_kind)
    b = to_operand(B, b_used, mode, "act")
    return ops.call("pase_tc_gemm_tn", a.hi, a.lo, lda, pitchA, offA, b.hi, b.lo, ldb, pitchB,
                    b_used // ldb, C, ldc, I, J, groups, rows, 1.0, a.alpha, 0, mode)


def tc_shapes_ok(lda, K, ldb):
    """True when gemm_nt would take the tensor-core path in the current mode."""
    mode = _MODES[PRECISION]
    esz = 2 if mode in (2, 3) else 4
    return mode is not None and lda % _eb(mode) == 0 and (K * esz) % 16 == 0 and \
        (ldb * esz) % 16 == 0


def _rows_ld(x):
    """(rows, cols) fp32 tensor with unit inner stride -> (flat view at its first element, ld)."""
    assert x.dim() == 2 and x.dtype == torch.float32, (x.shape, x.dtype)
    if x.stride(1) != 1 or (x.shape[0] > 1 and x.stride(0) % 4 != 0) or x.storage_offset() % 4 != 0:
        x = x.contiguous()
        if x.shape[1] % 4 != 0:
            pad = torch.zeros(x.shape[0], _ru4(x.shape[1]), dtype=x.dtype, device=x.device)
            pad[:, :x.shape[1]] = x
            x = pad[:, :x.shape[1]]
    ld = x.stride(0) if x.shape[0] > 1 else _ru4(x.shape[1])
    if ld % 4 != 0:
        pad = torch.zeros(x.shape[0], _ru4(x.shape[1]), dtype=x.dtype, device=x.device)
        pad[:, :x.shape[1]] = x
        x, ld = pad[:, :x.shape[1]], pad.stride(0)
    return x, ld


def _flat_from(x):
    """1-D view of x's storage starting at x's first element (base-pointer semantics)."""
    st = x.untyped_storage()
    n = st.nbytes() // 4 - x.storage_offset()
    return torch.as_strided(x, (n,), (1,), x.storage_offset())


class _LinearRows(torch.autograd.Function):
    """Y[rows, :N] = X[rows, :K] @ W[N, K]^T + b   (1x1 Conv1d / Linear on channel-last rows;
    minions.py:494-524, modules.py:543-556).  Y has ld = roundup(N, 4), padding zeroed."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x, ldx = _rows_ld(x.detach())
        rows, K = x.shape
        N = weight.shape[0]
        w2 = weight.detach().reshape(N, -1)
        assert w2.shape[1] == K and K % 4 == 0, "in-features %d must match and be a multiple of 4" % K
        w2 = w2.contiguous()
        ldo = _pad_ld(N)
        # +64 floats of slack: the tensor-core weight-gradient kernel reads whole 128-byte
        # column blocks of dY (DESIGN.md 4)
        buf = torch.empty(rows * ldo + 64, dtype=torch.float32, device=x.device)
        out = buf[:rows * ldo].view(rows, ldo)
        buf[rows * ldo:].zero_()
        if ldo != N:
            out[:, N:].zero_()
        # the input is a GEMM operand twice (A here, B of the weight-gradient GEMM in
        # backward): convert it to the operand format once and keep it
        xop = _flat_from(x)
        mode = _MODES[PRECISION]
        if mode not in (None, 0) and tc_shapes_ok(ldx, K, K):
            xop = to_operand(xop, rows * ldx, mode, "act")
        gemm_nt(xop, ldx, rows * ldx, w2.reshape(-1), K, N * K, out.reshape(-1), ldo,
                rows, N, K, None if bias is None else bias.detach().reshape(-1))
        ctx.save_for_backward(x, w2)
        ctx.xop = xop if isinstance(xop, Operand) else None
        ctx.ldx, ctx.N, ctx.has_bias, ctx.wshape, ctx.ldo = ldx, N, bias is not None, \
            weight.shape, ldo
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w2 = ctx.saved_tensors
        rows, K = x.shape
        N, ldx, ldo = ctx.N, ctx.ldx, ctx.ldo
        assert dy.shape == (rows, ldo)
        dev = x.device
        mode = _MODES[PRECISION]
        # the tensor-core weight-gradient kernel reads dY in whole 128-byte column blocks: a dY
        # whose leading dimension is a multiple of that block (every tensor-core mode pads so)
        # needs no slack; otherwise copy it into a buffer with 64 zeroed floats behind it
        blk = _eb(mode) if mode is not None else 4
        if dy.is_contiguous() and ldo % blk == 0 and dy.data_ptr() % 16 == 0:
            dyb = dy.reshape(-1)
            n_dy = rows * ldo
        else:
            dyb = torch.empty(rows * ldo + 64, dtype=torch.float32, device=dev)
            dyb[:rows * ldo].view(rows, ldo).copy_(dy)
            dyb[rows * ldo:].zero_()
            n_dy = rows * ldo + 64
        dyf = dyb
        # dY feeds both backward GEMMs: convert it to the operand format once
        if mode is not None and mode != 0 and tc_shapes_ok(ldo, ldo, ldo) and \
                ldx % _eb(mode) == 0 and K % _eb(mode) == 0 and ldo % 4 == 0:
            dyf = to_operand(dyb, n_dy, mode, "grad")
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            wT = torch.empty(K, ldo, dtype=torch.float32, device=dev)
            ops.call("pase_transpose_pad", w2.reshape(-1), K, wT.reshape(-1), ldo, N, K)
            dx = torch.empty(rows, K, dtype=torch.float32, device=dev)
            gemm_nt(dyf, ldo, rows * ldo, wT.reshape(-1), ldo, K * ldo, dx.reshape(-1), K,
                    rows, K, ldo, None, a_kind="grad")
        if ctx.needs_input_grad[1]:
            dWp = torch.empty(ldo, K, dtype=torch.float32, device=dev)
            xb = _flat_from(x)
            if ctx.xop is not None and isinstance(dyf, Operand):
                xb = ctx.xop                     # same format as the B operand of the TN GEMM
            gemm_tn(dyf, ldo, rows * ldo, xb, ldx, rows * ldx, dWp.reshape(-1), K,
                    ldo, K, rows)
            dW = dWp[:N].reshape(ctx.wshape)
        dy = dyb[:rows * ldo].view(rows, ldo)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            acc = torch.zeros(ldo, dtype=torch.float64, device=dev)
            ops.call("pase_colsum", dy.reshape(-1), ldo, rows, ldo, acc)
            dbf = torch.empty(ldo, dtype=torch.float32, device=dev)
            ops.call("pase_cast_d2f", acc, dbf, ldo, 1.0)
            db = dbf[:N]
        return dx, dW, db


def linear_rows(x, weight, bias=None):
    return _LinearRows.apply(x, weight, bias)


class _PReLURows(torch.autograd.Function):
    """Per-channel PReLU on (rows, ld) with C valid columns (modules.py:550, 111-113)."""

    @staticmethod
    def forward(ctx, u, alpha, C):
        u = u.detach()
        rows, ld = u.shape
        h = torch.empty_like(u)
        if ld != C:
            h[:, C:].zero_()
        ops.call("pase_prelu_fwd", u.reshape(-1), h.reshape(-1), alpha.detach().reshape(-1), rows,
                 C, ld, ld)
        ctx.save_for_backward(u, alpha.detach())
        ctx.C = C
        return h

    @staticmethod
    def backward(ctx, dh):
        u, alpha = ctx.saved_tensors
        rows, ld = u.shape
        C = ctx.C
        dh = dh.contiguous()
        du = torch.empty_like(u)
        if ld != C:
            du[:, C:].zero_()
        acc = torch.zeros(C, dtype=torch.float64, device=u.device)
        ops.call("pase_prelu_bwd", u.reshape(-1), dh.reshape(-1), alpha.reshape(-1), du.reshape(-1),
                 acc, rows, C, ld, ld, ld)
        da = torch.empty(C, dtype=torch.float32, device=u.device)
        ops.call("pase_cast_d2f", acc, da, C, 1.0)
        return du, da.view_as(alpha), None


def prelu_rows(u, alpha, C):
    return _PReLURows.apply(u, alpha, C)


class _TimeMean(torch.autograd.Function):
    """(B*T, C) rows -> (B, C): mean over time (GIM, cls_minions.py:96)."""

    @staticmethod
    def forward(ctx, x, B, T):
        x, ldx = _rows_ld(x.detach())
        C = x.shape[1]
        out = torch.empty(B, C, dtype=torch.float32, device=x.device)
        ops.call("pase_time_mean_fwd", _flat_from(x), ldx, out.reshape(-1), C, B, T, C)
        ctx.B, ctx.T, ctx.C = B, T, C
        return out

    @staticmethod
    def backward(ctx, dout):
        B, T, C = ctx.B, ctx.T, ctx.C
        dout = dout.contiguous()
        dx = torch.empty(B * T, C, dtype=torch.float32, device=dout.device)
        ops.call("pase_time_mean_bwd", dout.reshape(-1), C, dx.reshape(-1), C, B, T, C, 0)
        return dx, None, None


def time_mean_rows(x, B, T):
    return _TimeMean.apply(x, B, T)


class _NctToRows(torch.autograd.Function):
    """(B,C,T) -> (B*T, C) channel-last rows (boundary conversion for tensors that did not
    come from the encoder's channel-last output)."""

    @staticmethod
    def forward(ctx, x):
        x = x.detach().contiguous().float()
        B, C, T = x.shape
        out = torch.empty(B * T, C, dtype=torch.float32, device=x.device)
        ops.call("pase_nct_to_ntc", x.reshape(-1), out.reshape(-1), B, C, T, C)
        ctx.shape = (B, C, T)
        return out

    @staticmethod
    def backward(ctx, g):
        B, C, T = ctx.shape
        g = g.contiguous()
        dx = torch.empty(B, C, T, dtype=torch.float32, device=g.device)
        ops.call("pase_ntc_to_nct", g.reshape(-1), C, dx.reshape(-1), B, C, T)
        return dx


def nct_to_rows(x):
    return _NctToRows.apply(x)


class _FusedLinearCtxMSE(torch.autograd.Function):
    """Output layer of a regression head FUSED with its contextualised MSE (MLPMinion.W +
    ContextualizedLoss, minions.py:494-524, losses.py:15-37): loss = mean((h W^T + b -
    ctx_r(label))^2) without ever storing the (rows, F*r) prediction in fp32 -- the GEMM
    epilogue emits the fp16 pair of the (power-of-two scaled) residual, which IS the operand
    of the two backward GEMMs, plus sum residual^2 and the bias gradient's column sums.
    3xF16 precision only (the caller falls back to the unfused path otherwise)."""

    _buffers = {}

    @staticmethod
    def forward(ctx, h, weight, bias, label, F, r):
        h, ldh = _rows_ld(h.detach())
        rows, K = h.shape
        N = weight.shape[0]
        dev = h.device
        label = label.detach().contiguous().float()
        B, Fl, T = label.shape
        assert Fl == F and N == F * r and rows == B * T
        w2 = weight.detach().reshape(N, -1).contiguous()
        ldr = _ru(N, 128)
        hop = to_operand(_flat_from(h), rows * ldh, 3, "act")
        wop = to_operand(w2.reshape(-1), N * K, 3, "weight")
        # power-of-two scale from the bound |residual| <= max||h_m|| max||W_n|| + max|b| + max|label|
        am = torch.zeros(4, dtype=torch.float32, device=dev)
        ops.call("pase_rownorm_max", _flat_from(h), ldh, rows, K, am[0:1])
        ops.call("pase_rownorm_max", w2.reshape(-1), K, N, K, am[1:2])
        if bias is not None:
            ops.call("pase_absmax", bias.detach().reshape(-1), N, am[2:3])
        ops.call("pase_absmax", label.reshape(-1), label.numel(), am[3:4])
        scale = torch.empty(2, dtype=torch.float32, device=dev)
        ops.call("pase_bound_scale", am, scale)
        # persistent residual buffers (two lps heads of the same shape are alive at once)
        pool = _FusedLinearCtxMSE._buffers.setdefault((rows, ldr, str(dev)), [])
        ent = next((e for e in pool if not e["busy"]), None)
        if ent is None:
            ent = {"hi": torch.zeros(rows * ldr, dtype=torch.float16, device=dev),
                   "lo": torch.zeros(rows * ldr, dtype=torch.float16, device=dev), "busy": False}
            pool.append(ent)
        ent["busy"] = True                        # released by backward
        acc = torch.zeros(1 + ldr, dtype=torch.float64, device=dev)
        ops.call("pase_tc_gemm_nt_ctxmse", hop.hi, hop.lo, rows, ldh, wop.hi, wop.lo, K,
                 ent["hi"], ent["lo"], ldr, rows, N, K,
                 None if bias is None else bias.detach().reshape(-1), label.reshape(-1),
                 B, F, T, r, scale, acc[0:1], acc[1:])
        ctx.save_for_backward(h, w2, scale, acc)
        ctx.hop, ctx.ent = hop, ent
        ctx.dims = (rows, K, N, ldr, ldh, weight.shape, bias is not None)
        return _loss_scalar(acc[0:1], rows * N)

    @staticmethod
    def backward(ctx, g):
        h, w2, scale, acc = ctx.saved_tensors
        rows, K, N, ldr, ldh, wshape, has_bias = ctx.dims
        ent, dev = ctx.ent, h.device
        coef = 2.0 / float(rows * N)
        # d loss / d pred = g * coef * residual; the stored pair is s * residual
        adev = (g.detach().reshape(1).float() * coef) * scale[0:1]
        rop = Operand(ent["hi"], ent["lo"], adev)
        dh = dW = db = None
        if ctx.needs_input_grad[0]:
            wT = torch.empty(K, ldr, dtype=torch.float32, device=dev)
            ops.call("pase_transpose_pad", w2.reshape(-1), K, wT.reshape(-1), ldr, N, K)
            dh = torch.empty(rows, K, dtype=torch.float32, device=dev)
            gemm_nt(rop, ldr, rows * ldr, wT.reshape(-1), ldr, K * ldr, dh.reshape(-1), K,
                    rows, K, ldr, None, a_kind="grad")
        if ctx.needs_input_grad[1]:
            dWp = torch.empty(ldr, K, dtype=torch.float32, device=dev)
            gemm_tn(rop, ldr, rows * ldr, ctx.hop, ldh, rows * ldh, dWp.reshape(-1), K, ldr, K, rows)
            dW = dWp[:N].reshape(wshape)
        if has_bias and ctx.needs_input_grad[2]:
            dbf = torch.empty(ldr, dtype=torch.float32, device=dev)
            ops.call("pase_cast_d2f", acc[1:], dbf, ldr, coef)
            db = dbf[:N] * g.detach().float()
        ent["busy"] = False
        return dh, dW, db, None, None, None


def fused_linear_ctx_mse(h, weight, bias, label, F, r):
    return _FusedLinearCtxMSE.apply(h, weight, bias, label, F, r)


def fused_head_ok(K, ldh):
    """The fused output layer needs the 3xF16 tensor-core path."""
    return _MODES[PRECISION] == 3 and ldh % 64 == 0 and K % 64 == 0


# ------------------------------------------------------------------ losses ---
def _loss_scalar(acc, numel):
    return (acc / float(numel)).float().reshape(())


class _CtxMSE(torch.autograd.Function):
    """mean((pred - contextualise_r(label))^2) on channel-last predictions without
    materialising the r-times unfolded label (losses.py:15-37 + nn.MSELoss)."""

    @staticmethod
    def forward(ctx, pred, label, F, r):
        pred = pred.detach()
        rows, ldp = pred.shape
        label = label.detach().contiguous().float()
        B, Fl, T = label.shape
        assert Fl == F and rows == B * T, (label.shape, pred.shape)
        acc = torch.zeros(1, dtype=torch.float64, device=pred.device)
        ops.call("pase_ctx_mse_fwd", pred.reshape(-1), ldp, label.reshape(-1), B, F, T, r, acc)
        ctx.save_for_backward(pred, label)
        ctx.dims = (B, F, T, r, ldp)
        return _loss_scalar(acc, rows * F * r)

    @staticmethod
    def backward(ctx, g):
        pred, label = ctx.saved_tensors
        B, F, T, r, ldp = ctx.dims
        dpred = torch.empty_like(pred)
        if ldp != F * r:
            dpred[:, F * r:].zero_()
        ops.call("pase_ctx_mse_bwd", pred.reshape(-1), ldp, label.reshape(-1), B, F, T, r,
                 2.0 / float(B * T * F * r), g.detach().reshape(-1).float(), dpred.reshape(-1), ldp)
        return dpred, None, None, None


def ctx_mse_rows(pred, label, F, r):
    return _CtxMSE.apply(pred, label, F, r if r is not None else 1)


class _L1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        pred, target = pred.detach().contiguous(), target.detach().contiguous().float()
        assert pred.numel() == target.numel()
        acc = torch.zeros(1, dtype=torch.float64, device=pred.device)
        ops.call("pase_l1_fwd", pred.reshape(-1), target.reshape(-1), pred.numel(), acc)
        ctx.save_for_backward(pred, target)
        return _loss_scalar(acc, pred.numel())

    @staticmethod
    def backward(ctx, g):
        pred, target = ctx.saved_tensors
        d = torch.empty_like(pred)
        ops.call("pase_l1_bwd", pred.reshape(-1), target.reshape(-1), pred.numel(),
                 1.0 / float(pred.numel()), g.detach().reshape(-1).float(), d.reshape(-1))
        return d, None


def l1_loss(pred, target):
    return _L1.apply(pred, target)


class _BCEPairs(torch.autograd.Function):
    """BCEWithLogits against [ones; zeros] (make_labels, cls_minions.py:47-51)."""

    @staticmethod
    def forward(ctx, logit, n_pos):
        logit = logit.detach().contiguous()
        acc = torch.zeros(1, dtype=torch.float64, device=logit.device)
        ops.call("pase_bce_pairs_fwd", logit.reshape(-1), logit.numel(), n_pos, acc)
        ctx.save_for_backward(logit)
        ctx.n_pos = n_pos
        return _loss_scalar(acc, logit.numel())

    @staticmethod
    def backward(ctx, g):
        (logit,) = ctx.saved_tensors
        d = torch.empty_like(logit)
        ops.call("pase_bce_pairs_bwd", logit.reshape(-1), logit.numel(), ctx.n_pos,
                 1.0 / float(logit.numel()), g.detach().reshape(-1).float(), d.reshape(-1))
        return d, None


def bce_pairs(logit, n_pos):
    return _BCEPairs.apply(logit, n_pos)
