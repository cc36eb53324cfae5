"""Differentiable building blocks of the worker heads over the C-ABI kernels.

Tensors are channel-last "row" matrices (rows = sample*time, columns =
channels) with a leading dimension that is a multiple of 4 floats; padding
columns are kept at zero so a padded matrix can be fed straight back as a GEMM
operand.  Each autograd Function launches only kernels of pase_b200/csrc.
"""
import os

import torch

from . import gemm, ops

# GEMM numerics of the heads (same meaning as WaveFe.precision): "3xf16" / "3xtf32" (wgmma,
# fp32-equivalent products), "tf32", "bf16" (bf16 operands, fp32 everything else), or "fp32"
# (FFMA kernels).
PRECISION = os.environ.get("PASE_B200_PRECISION", "3xf16")


def set_precision(p):
    global PRECISION
    if p not in gemm.PRECISIONS:
        raise ValueError("precision must be one of %s" % sorted(gemm.PRECISIONS))
    PRECISION = p


def gemm_precision():
    """The heads' precision record (gemm.PRECISIONS)."""
    return gemm.PRECISIONS[PRECISION]


_F16X3 = gemm.PRECISIONS["3xf16"]          # the fused regression head's only format


def _ru4(n):
    return (n + 3) // 4 * 4


def _ru(n, m):
    return (n + m - 1) // m * m


def _pad_ld(n):
    """leading dimension of a rows-matrix with n columns: tensor-core modes pad to one
    128-byte row so the matrix can itself be a TMA operand."""
    p = gemm_precision()
    return _ru(n, p.eb) if p.tc else _ru4(n)


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
        p, xf = gemm_precision(), _flat_from(x)
        xop = gemm.to_operand(p, xf, rows * ldx) if gemm.nt_ok(p, ldx, K, K) else None
        gemm.nt(p, xf, ldx, rows * ldx, w2.reshape(-1), K, out.reshape(-1), ldo, rows, N, K,
                bias=None if bias is None else bias.detach().reshape(-1), a_op=xop)
        ctx.save_for_backward(x, w2)
        ctx.xop = xop
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
        p = gemm_precision()
        # the tensor-core weight-gradient kernel reads dY in whole 128-byte column blocks: a dY
        # whose leading dimension is a multiple of that block (every tensor-core mode pads so)
        # needs no slack; otherwise copy it into a buffer with 64 zeroed floats behind it
        blk = p.eb if p.tc else 4
        if dy.is_contiguous() and ldo % blk == 0 and dy.data_ptr() % 16 == 0:
            dyb = dy.reshape(-1)
            n_dy = rows * ldo
        else:
            dyb = torch.empty(rows * ldo + 64, dtype=torch.float32, device=dev)
            dyb[:rows * ldo].view(rows, ldo).copy_(dy)
            dyb[rows * ldo:].zero_()
            n_dy = rows * ldo + 64
        # dY feeds both backward GEMMs: when both take the tensor cores, convert it to the
        # operand format once (and the weight gradient reuses the forward's operand of X)
        dyop = None
        if gemm.nt_ok(p, ldo, ldo, ldo) and gemm.tn_ok(p, ldo, ldx, ldo, K):
            dyop = gemm.to_operand(p, dyb, n_dy, "grad")
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            wT = torch.empty(K, ldo, dtype=torch.float32, device=dev)
            ops.call("pase_transpose_pad", w2.reshape(-1), K, wT.reshape(-1), ldo, N, K)
            dx = torch.empty(rows, K, dtype=torch.float32, device=dev)
            gemm.nt(p, dyb, ldo, rows * ldo, wT.reshape(-1), ldo, dx.reshape(-1), K, rows, K,
                    ldo, a_kind="grad", a_op=dyop)
        if ctx.needs_input_grad[1]:
            dWp = torch.empty(ldo, K, dtype=torch.float32, device=dev)
            gemm.tn(p, dyb, ldo, rows * ldo, _flat_from(x), ldx, rows * ldx, dWp.reshape(-1), K,
                    ldo, K, rows, a_op=dyop, b_op=None if dyop is None else ctx.xop)
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


def check_spc_frames(T, N, seq_pad, t, future_t, past_t):
    """The ranges SPCMinion draws from (minions.py:609-627): refuse indices outside them before
    they reach the device, where the gather kernels trust them."""
    M = seq_pad + N
    if not (M + 1 <= t < T - M and t + seq_pad <= future_t < T - N and
            N <= past_t < t - seq_pad):
        raise ValueError("SPC frames (t=%r, future_t=%r, past_t=%r) outside the ranges of T'=%d "
                         "frames, N=%d, seq_pad=%d: need %d <= t < %d, t + %d <= future_t < %d, "
                         "%d <= past_t < t - %d" % (t, future_t, past_t, T, N, seq_pad, M + 1,
                                                    T - M, seq_pad, T - N, N, seq_pad))


class _SPCGather(torch.autograd.Function):
    """(B*T, C) rows -> (2B, (N+1)*C) rows [cur | fut ; cur | past] of the SPC worker, the three
    frame indices read from the device int64 tensor `frames` {t, future_t, past_t}."""

    @staticmethod
    def forward(ctx, x, frames, B, T, N, seq_pad):
        x = x.detach()
        C = x.shape[1]
        if x.stride(1) != 1:
            x = x.contiguous()
        ldx = x.stride(0) if x.shape[0] > 1 else C
        out = torch.empty(2 * B, (N + 1) * C, dtype=torch.float32, device=x.device)
        ops.call("pase_spc_gather", x, ldx, frames, B, T, C, N, seq_pad, out)
        ctx.save_for_backward(frames)
        ctx.dims = (B, T, C, N, seq_pad)
        return out

    @staticmethod
    def backward(ctx, g):
        (frames,) = ctx.saved_tensors
        B, T, C, N, seq_pad = ctx.dims
        g = g.contiguous()
        dx = torch.empty(B * T, C, dtype=torch.float32, device=g.device)
        ops.call("pase_spc_gather_bwd", g, frames, B, T, C, N, seq_pad, dx)
        return dx, None, None, None, None, None


def spc_gather(rows, B, T, N, seq_pad, frames):
    """SPC input rows of the (B*T, C) encoder rows.  frames: a device int64 tensor of
    {t, future_t, past_t} (trusted: a captured step's table, filled by a planner that checked
    it), or a host triple, checked here and uploaded."""
    if not isinstance(frames, torch.Tensor):
        check_spc_frames(T, N, seq_pad, *frames)
        src = torch.tensor([int(f) for f in frames], dtype=torch.int64)
        if rows.is_cuda:
            src = src.pin_memory()
        frames = src.to(rows.device, non_blocking=True)
    return _SPCGather.apply(rows, frames, B, T, N, seq_pad)


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
    3xF16 precision only (the caller falls back to the unfused path otherwise).

    ``need_grad`` False (a validation pass): the loss-only epilogue, which writes sum
    residual^2 and nothing else -- no residual pair, no pool entry, nothing saved."""

    _buffers = {}

    @staticmethod
    def forward(ctx, h, weight, bias, label, F, r, need_grad):
        h, ldh = _rows_ld(h.detach())
        rows, K = h.shape
        N = weight.shape[0]
        dev = h.device
        label = label.detach().contiguous().float()
        B, Fl, T = label.shape
        assert Fl == F and N == F * r and rows == B * T
        w2 = weight.detach().reshape(N, -1).contiguous()
        ldr = _ru(N, 128)
        hop = gemm.to_operand(_F16X3, _flat_from(h), rows * ldh)
        wop = gemm.to_operand(_F16X3, w2.reshape(-1), N * K, "weight")
        b = None if bias is None else bias.detach().reshape(-1)
        if not need_grad:
            acc = torch.zeros(1, dtype=torch.float64, device=dev)
            ops.call("pase_tc_gemm_nt_ctxmse", hop.hi, hop.lo, rows, ldh, wop.hi, wop.lo, K,
                     None, None, ldr, rows, N, K, b, label.reshape(-1), B, F, T, r, None, acc,
                     None)
            return _loss_scalar(acc, rows * N)
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
                 ent["hi"], ent["lo"], ldr, rows, N, K, b, label.reshape(-1),
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
        rop = gemm.Operand(ent["hi"], ent["lo"], adev)      # exists only as the fp16 pair
        dh = dW = db = None
        if ctx.needs_input_grad[0]:
            wT = torch.empty(K, ldr, dtype=torch.float32, device=dev)
            ops.call("pase_transpose_pad", w2.reshape(-1), K, wT.reshape(-1), ldr, N, K)
            dh = torch.empty(rows, K, dtype=torch.float32, device=dev)
            gemm.nt(_F16X3, None, ldr, rows * ldr, wT.reshape(-1), ldr, dh.reshape(-1), K,
                    rows, K, ldr, a_kind="grad", a_op=rop)
        if ctx.needs_input_grad[1]:
            dWp = torch.empty(ldr, K, dtype=torch.float32, device=dev)
            gemm.tn(_F16X3, None, ldr, rows * ldr, None, ldh, rows * ldh, dWp.reshape(-1), K,
                    ldr, K, rows, a_op=rop, b_op=ctx.hop)
            dW = dWp[:N].reshape(wshape)
        if has_bias and ctx.needs_input_grad[2]:
            dbf = torch.empty(ldr, dtype=torch.float32, device=dev)
            ops.call("pase_cast_d2f", acc[1:], dbf, ldr, coef)
            db = dbf[:N] * g.detach().float()
        ent["busy"] = False
        return dh, dW, db, None, None, None, None


def fused_linear_ctx_mse(h, weight, bias, label, F, r):
    # only backward releases a residual pair: without one to come (no_grad, or nothing that
    # requires grad) the forward must not take a pair
    need_grad = torch.is_grad_enabled() and any(
        t is not None and t.requires_grad for t in (h, weight, bias))
    return _FusedLinearCtxMSE.apply(h, weight, bias, label, F, r, need_grad)


def fused_head_ok(K, ldh):
    """The fused output layer needs the 3xF16 tensor-core path."""
    return gemm_precision() is _F16X3 and ldh % 64 == 0 and K % 64 == 0


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
