"""The shared helpers of the emulation (strided views, reflect indices, operand formats) and
the entry points of uniform shape: the GEMMs, BatchNorm/PReLU, QRNN, SincNet, losses, casts and
weight re-layouts."""
import math
import torch

# select_output mode of the output entry points' `mode` argument
_MODES = {0: None, 1: "avg_norm", 2: "avg_concat", 3: "avg_norm_concat"}


def _as(buf, size, stride, offset=0):
    return torch.as_strided(buf, size, stride, buf.storage_offset() + offset)


def _rows(tab, n, width):
    """The first n rows of a job table of `width` columns, as lists."""
    return tab[:n * width].view(n, width).tolist()


def _reflect(idx, T):
    idx = idx.abs()
    return torch.where(idx >= T, 2 * (T - 1) - idx, idx)


def pase_gemm_nt(A, lda, B, ldb, C, ldc, M, N, K, alpha, bias, rows_in, t_valid, rows_out,
                 fold, colsum, colsumsq, accumulate):
    a = _as(A, (M, K), (lda, 1)).double()
    b = _as(B, (N, K), (ldb, 1)).double()
    out = (a @ b.t()) * alpha
    if bias is not None:
        out = out + bias[:N].double()[None, :]
    out = out.float()
    m = torch.arange(M)
    g, u = m // rows_in, m % rows_in
    keep = (u * fold) < t_valid                       # rows with at least one valid column
    m, g, u, out = m[keep], g[keep], u[keep], out[keep]
    cpf = N // fold
    valid = (u[:, None] * fold + (torch.arange(N) // cpf)[None, :]) < t_valid
    orow = g * rows_out + u
    nrows = int(orow.max()) + 1
    Cv = _as(C, (nrows, N), (ldc, 1))
    cur = Cv[orow]
    if accumulate:
        out = out + cur
    Cv[orow] = torch.where(valid, out, cur)
    if colsum is not None:
        ov = torch.where(valid, out, torch.zeros_like(out)).double()
        colsum[:N] += ov.sum(0)
        colsumsq[:N] += (ov * ov).sum(0)


def pase_gemm_tn(A, lda, pitchA, offA, B, ldb, pitchB, offB, C, ldc, I, J, groups,
                 rows_per_group, alpha, accumulate):
    r = torch.arange(groups * rows_per_group)
    g, u = r // rows_per_group, r % rows_per_group
    ra, rb = g * pitchA + offA + u, g * pitchB + offB + u
    a = _as(A, (int(ra.max()) + 1, I), (lda, 1))[ra].double()
    b = _as(B, (int(rb.max()) + 1, J), (ldb, 1))[rb].double()
    out = ((a.t() @ b) * alpha).float()
    Cv = _as(C, (I, J), (ldc, 1))
    if accumulate:
        Cv += out
    else:
        Cv.copy_(out)


def pase_conv_w_to_fwd(W, Wt, Cout, Cin, k):
    Wt[:Cout * Cin * k] = W[:Cout * Cin * k].view(Cout, Cin, k).permute(0, 2, 1).reshape(-1)


def pase_conv_w_from_fwd(dWt, dW, Cout, Cin, k):
    dW[:Cout * Cin * k] = dWt[:Cout * Cin * k].view(Cout, k, Cin).permute(0, 2, 1).reshape(-1)


def pase_conv_w_to_dgrad(W, Wd, Cout, Cin, k, s, taps):
    w = W[:Cout * Cin * k].view(Cout, Cin, k)
    wp = torch.zeros(Cout, Cin, taps * s)
    wp[:, :, :k] = w
    wp = wp.view(Cout, Cin, taps, s).flip(2)            # [co, ci, v, p], tap = s*(taps-1-v)+p
    Wd[:s * Cin * taps * Cout] = wp.permute(3, 1, 2, 0).reshape(-1)


def pase_deconv_w_to_fwd(W, Wu, Cin, Cout, k, s, taps):
    w = W[:Cin * Cout * k].view(Cin, Cout, k)
    wp = torch.zeros(Cin, Cout, taps * s)
    wp[:, :, :k] = w
    wp = wp.view(Cin, Cout, taps, s).flip(2)            # [ci, co, v, p]
    Wu[:s * Cout * taps * Cin] = wp.permute(3, 1, 2, 0).reshape(-1)


def pase_deconv_w_from_fwd(dWu, dW, Cin, Cout, k, s, taps):
    g = dWu[:s * Cout * taps * Cin].view(s, Cout, taps, Cin).permute(3, 1, 2, 0)  # ci,co,v,p
    g = g.flip(2).reshape(Cin, Cout, taps * s)[:, :, :k]
    dW[:Cin * Cout * k] = g.reshape(-1)


def pase_deconv_w_to_bwd(W, Wb, Cin, Cout, k):
    Wb[:Cin * Cout * k] = W[:Cin * Cout * k].view(Cin, Cout, k).permute(0, 2, 1).reshape(-1)


def pase_transpose_pad(src, lds, dst, ldd, rows, cols):
    s = _as(src, (rows, cols), (lds, 1))
    d = _as(dst, (cols, ldd), (ldd, 1))
    d.zero_()
    d[:, :rows] = s.t()


def _sinc_filters(low_hz, band_hz, n_, win, C, k, min_low, min_band, sr):
    low = min_low + low_hz[:C].abs().view(-1, 1)
    high = torch.clamp(low + min_band + band_hz[:C].abs().view(-1, 1), min_low, sr / 2)
    band = (high - low)[:, 0]
    n = n_.view(1, -1)
    left = (torch.sin(high @ n) - torch.sin(low @ n)) / (n / 2) * win.view(1, -1)
    bp = torch.cat([left, 2 * band.view(-1, 1), left.flip(1)], 1)
    return bp / (2 * band[:, None])


def pase_sinc_make(low_hz, band_hz, n_, win, filt, Wp, C, k, fold, Kv, min_low, min_band, sr):
    f = _sinc_filters(low_hz, band_hz, n_, win, C, k, min_low, min_band, sr)
    if filt is not None:
        filt[:C * k] = f.reshape(-1)
    W = torch.zeros(fold, C, Kv)
    for p in range(fold):
        W[p, :, p:p + k] = f
    Wp[:fold * C * Kv] = W.reshape(-1)


def pase_sinc_grad(dWp, low_hz, band_hz, n_, win, dlow, dband, C, k, fold, Kv, min_low,
                   min_band, sr):
    l = low_hz[:C].detach().clone().requires_grad_(True)
    b = band_hz[:C].detach().clone().requires_grad_(True)
    f = _sinc_filters(l, b, n_, win, C, k, min_low, min_band, sr)
    g = dWp[:fold * C * Kv].view(fold, C, Kv)
    df = sum(g[p, :, p:p + k] for p in range(fold))
    gl, gb = torch.autograd.grad((f * df).sum(), [l, b])
    dlow[:C] = gl
    dband[:C] = gb


F16_LO_MUL = 2048.0        # lo' = rn_f16((x - hi) * 2^11)


def _store_fmt(val, dst, dst_lo, fmt, size, stride):
    """Write fp32 `val` (shape `size`) into the strided view of dst in storage format `fmt`
    (0 fp32 [+ tf32 residual], 1 bf16, 2 fp16 pair); returns the value a reader sees."""
    if fmt == 0:
        _as(dst, size, stride).copy_(val)
        if dst_lo is not None:
            _as(dst_lo, size, stride).copy_(_residual(val.contiguous()))
        return val
    if fmt == 1:
        assert dst.dtype == torch.bfloat16
        _as(dst, size, stride).copy_(val.to(torch.bfloat16))
        return val.to(torch.bfloat16).float()
    assert dst.dtype == torch.float16 and dst_lo.dtype == torch.float16
    hi = val.to(torch.float16)
    _as(dst, size, stride).copy_(hi)
    _as(dst_lo, size, stride).copy_(((val - hi.float()) * F16_LO_MUL).to(torch.float16))
    return val


def f16_grad_scale(bound):
    """power of two s with bound * s <= 2^14 (common.cuh::f16_grad_scale)."""
    bound = float(bound)
    if not (bound > 0.0) or not (bound < 3.0e38):
        return 1.0
    _, e = math.frexp(bound)
    k = max(-100, min(100, 14 - e))
    return math.ldexp(1.0, k)


def pase_reflect_pad_wave(x, dst, dst_lo, dst_fmt, N, T, padL, padR, pitch):
    Tp = T + padL + padR
    src = x[:N * T].view(N, T)
    idx = _reflect(torch.arange(Tp) - padL, T)
    _store_fmt(src[:, idx], dst, dst_lo, dst_fmt, (N, Tp), (pitch, 1))


def pase_cast_bf16(x, dst, n):
    dst[:n] = x[:n].to(torch.bfloat16)


def pase_absmax(x, n, amax):
    amax[0] = max(float(amax[0]), float(x[:n].abs().max()))


def pase_split_f16(x, hi, lo, n, amax, scale_out):
    s = f16_grad_scale(float(amax[0]) * 1.0001) if amax is not None else 1.0
    if scale_out is not None:
        scale_out[0], scale_out[1] = 1.0 / s, s
    v = x[:n] * s
    h = v.to(torch.float16)
    hi[:n] = h
    lo[:n] = ((v - h.float()) * F16_LO_MUL).to(torch.float16)


def pase_bn_finalize(colsum, colsumsq, C, fold, count, gamma, beta, rm, rv, momentum, eps,
                     mean, invstd, scale, shift):
    s = colsum[:C * fold].view(fold, C).sum(0)
    q = colsumsq[:C * fold].view(fold, C).sum(0)
    m = s / count
    var = (q / count - m * m).clamp_min(0)
    is_ = 1.0 / torch.sqrt(var + eps)
    if rm is not None:
        unb = var * count / (count - 1) if count > 1 else var
        rm[:C] = ((1 - momentum) * rm[:C].double() + momentum * m).float()
        rv[:C] = ((1 - momentum) * rv[:C].double() + momentum * unb).float()
    g = gamma[:C].double() if gamma is not None else torch.ones(C, dtype=torch.float64)
    b = beta[:C].double() if beta is not None else torch.zeros(C, dtype=torch.float64)
    mean[:C] = m.float()
    invstd[:C] = is_.float()
    scale[:C] = (g * is_).float()
    shift[:C] = (b - m * g * is_).float()


def pase_bn_eval_affine(rm, rv, gamma, beta, C, eps, mean, invstd, scale, shift):
    is_ = 1.0 / torch.sqrt(rv[:C].double() + eps)
    g = gamma[:C].double() if gamma is not None else torch.ones(C, dtype=torch.float64)
    b = beta[:C].double() if beta is not None else torch.zeros(C, dtype=torch.float64)
    mean[:C] = rm[:C]
    invstd[:C] = is_.float()
    scale[:C] = (g * is_).float()
    shift[:C] = (b - rm[:C].double() * g * is_).float()


def _prelu(u, a):
    return torch.where(u > 0, u, a * u)


def _residual(a):
    return _tf32_rn(a - _tf32_trunc(a))


def pase_bn_prelu_pad_fwd(y, y_bf16, y_ss, N, T, C, scale, shift, alpha, dst, dst_lo, dst_fmt,
                          d_ss, d_rs, padL, padR, pool, p_ss, p_rs, pool_d, pool_T):
    assert (y.dtype == torch.bfloat16) == bool(y_bf16)
    yv = _as(y, (N, T, C), (y_ss, C, 1)).float()
    a = _prelu(yv * scale[:C] + shift[:C], alpha[:C])
    Tp = T + padL + padR
    idx = _reflect(torch.arange(Tp) - padL, T)
    seen = _store_fmt(a[:, idx], dst, dst_lo, dst_fmt, (N, Tp, C), (d_ss, d_rs, 1))
    if pool is not None and pool_d > 0:
        L = pool_T * pool_d
        pv = _as(pool, (N, pool_T, C), (p_ss, p_rs, 1))
        pv += seen[:, padL:padL + L].reshape(N, pool_T, pool_d, C).mean(2)


def _bwd_grad_sources(N, T, C, srcA, a_bf16, a_ss, a_rs, padL, padR, srcB, b_ss, b_rs, b_shift,
                      pool, p_ss, p_rs, pool_d, pool_T):
    g = torch.zeros(N, T, C)
    if srcA is not None:
        assert (srcA.dtype == torch.bfloat16) == bool(a_bf16)
        Tp = T + padL + padR
        av = _as(srcA, (N, Tp, C), (a_ss, a_rs, 1)).float()
        idx = _reflect(torch.arange(Tp) - padL, T)
        g.index_add_(1, idx, av.contiguous())
    if srcB is not None:
        bv = _as(srcB, (N, T, C), (b_ss, b_rs, 1))
        if b_shift >= 0:
            g[:, :T - b_shift] += bv[:, b_shift:]
        else:
            g[:, -b_shift:] += bv[:, :T + b_shift]
    if pool is not None and pool_d > 0:
        L = pool_T * pool_d
        pv = _as(pool, (N, pool_T, C), (p_ss, p_rs, 1))
        g[:, :L] += (pv / pool_d).repeat_interleave(pool_d, dim=1)
    return g


def pase_bn_prelu_bwd_reduce(y, y_bf16, y_ss, N, T, C, mean, invstd, scale, shift, alpha,
                             srcA, a_bf16, a_ss, a_rs, padL, padR, srcB, b_ss, b_rs, b_shift,
                             pool, p_ss, p_rs, pool_d, pool_T, dst, d_ss, S1, S2, dalpha, amax):
    assert (y.dtype == torch.bfloat16) == bool(y_bf16) and (dst is None or dst.dtype == y.dtype)
    yv = _as(y, (N, T, C), (y_ss, C, 1)).float()
    g = _bwd_grad_sources(N, T, C, srcA, a_bf16, a_ss, a_rs, padL, padR, srcB, b_ss, b_rs,
                          b_shift, pool, p_ss, p_rs, pool_d, pool_T)
    u = yv * scale[:C] + shift[:C]
    pos = u > 0
    du = torch.where(pos, g, alpha[:C] * g)
    xh = (yv - mean[:C]) * invstd[:C]
    S1[:C] += du.double().sum((0, 1))
    S2[:C] += (du * xh).double().sum((0, 1))
    dalpha[:C] += torch.where(pos, torch.zeros_like(g), u * g).double().sum((0, 1))
    if amax is not None:
        amax[0] = max(float(amax[0]), float(du.abs().max()))
        amax[1] = max(float(amax[1]), float(xh.abs().max()))
    if dst is not None:
        _as(dst, (N, T, C), (d_ss, C, 1)).copy_(du.to(dst.dtype))


def pase_bn_prelu_bwd_apply_src(y, y_bf16, y_ss, N, T, C, mean, invstd, gamma, scale, shift, alpha,
                                S1, S2, count, srcA, a_bf16, a_ss, a_rs, padL, padR, srcB, b_ss,
                                b_rs, b_shift, pool, p_ss, p_rs, pool_d, pool_T, dst, dst_lo,
                                dst_fmt, d_ss, dbias, amax, scale_out):
    assert (y.dtype == torch.bfloat16) == bool(y_bf16)
    yv = _as(y, (N, T, C), (y_ss, C, 1)).float()
    g = _bwd_grad_sources(N, T, C, srcA, a_bf16, a_ss, a_rs, padL, padR, srcB, b_ss, b_rs,
                          b_shift, pool, p_ss, p_rs, pool_d, pool_T)
    u = yv * scale[:C] + shift[:C]
    du = torch.where(u > 0, g, alpha[:C] * g)
    _bn_apply(y, y_bf16, y_ss, N, T, C, mean, invstd, gamma, S1, S2, count, du.reshape(-1), T * C,
              dst, dst_lo, dst_fmt, d_ss, dbias, amax, scale_out)


def pase_bn_prelu_bwd_apply(y, y_bf16, y_ss, N, T, C, mean, invstd, gamma, S1, S2, count, du,
                            dst, dst_lo, dst_fmt, d_ss, dbias, amax, scale_out):
    assert du.dtype == y.dtype
    _bn_apply(y, y_bf16, y_ss, N, T, C, mean, invstd, gamma, S1, S2, count, du, d_ss, dst, dst_lo,
              dst_fmt, d_ss, dbias, amax, scale_out)


def _bn_apply(y, y_bf16, y_ss, N, T, C, mean, invstd, gamma, S1, S2, count, du, du_ss, dst, dst_lo,
              dst_fmt, d_ss, dbias, amax, scale_out):
    """pase_bn_prelu_bwd_apply with du read at sample stride du_ss (fp32 when the caller
    computed it)."""
    assert (y.dtype == torch.bfloat16) == bool(y_bf16)
    yv = _as(y, (N, T, C), (y_ss, C, 1)).float()
    dv = _as(du, (N, T, C), (du_ss, C, 1)).float()
    xh = (yv - mean[:C]) * invstd[:C]
    gi = (gamma[:C] if gamma is not None else 1.0) * invstd[:C]
    m1, m2 = (S1[:C] / count).float(), (S2[:C] / count).float()
    out = gi * (dv - m1 - xh * m2)
    s = 1.0
    if dst_fmt == 2:
        gia = gi.abs() if isinstance(gi, torch.Tensor) else torch.full((C,), abs(gi))
        bound = float((gia * (float(amax[0]) + m1.abs() + float(amax[1]) * m2.abs())).max())
        s = f16_grad_scale(bound * 1.0001)
        scale_out[0], scale_out[1] = 1.0 / s, s
    _store_fmt(out * s, dst, dst_lo, dst_fmt, (N, T, C), (d_ss, C, 1))
    if dbias is not None:
        dbias[:C] += out.double().sum((0, 1))


def pase_prelu_fwd(u, h, alpha, rows, C, ldu, ldh):
    _as(h, (rows, C), (ldh, 1)).copy_(_prelu(_as(u, (rows, C), (ldu, 1)), alpha[:C]))


def pase_prelu_bwd(u, dh, alpha, du, dalpha, rows, C, ldu, lddh, lddu):
    uv, g = _as(u, (rows, C), (ldu, 1)), _as(dh, (rows, C), (lddh, 1))
    pos = uv > 0
    out = torch.where(pos, g, alpha[:C] * g)
    dalpha[:C] += torch.where(pos, torch.zeros_like(g), uv * g).double().sum(0)
    _as(du, (rows, C), (lddu, 1)).copy_(out)


def pase_colsum(X, ld, rows, C, acc):
    acc[:C] += _as(X, (rows, C), (ld, 1)).double().sum(0)


def pase_cast_d2f(src, dst, n, scale):
    dst[:n] = (src[:n] * scale).float()


def pase_out_affine_nct(y, scale, shift, out, out_ntc, N, T, C):
    # one rounding of y*scale + shift, as the kernel's fmaf
    v = (y[:N * T * C].view(N, T, C).double() * scale[:C].double() + shift[:C].double()).float()
    out[:N * C * T] = v.permute(0, 2, 1).reshape(-1)
    if out_ntc is not None:
        out_ntc[:N * T * C] = v.reshape(-1)


def pase_out_bwd_reduce(dout, dout_ntc, y, mean, invstd, N, T, C, g_ntc, S1, S2):
    g = torch.zeros(N, T, C)
    if dout is not None:
        g += dout[:N * C * T].view(N, C, T).permute(0, 2, 1)
    if dout_ntc is not None:
        g += dout_ntc[:N * T * C].view(N, T, C)
    xh = (y[:N * T * C].view(N, T, C) - mean[:C]) * invstd[:C]
    S1[:C] += g.double().sum((0, 1))
    S2[:C] += (g * xh).double().sum((0, 1))
    g_ntc[:N * T * C] = g.reshape(-1)


def pase_out_bwd_apply(g, y, mean, invstd, scale, S1, S2, count, use_stats, rows, C):
    gv = g[:rows * C].view(rows, C)
    v = gv
    if use_stats:
        xh = (y[:rows * C].view(rows, C) - mean[:C]) * invstd[:C]
        v = gv - (S1[:C] / count).float() - xh * (S2[:C] / count).float()
    gv.copy_(v * scale[:C])


def pase_nct_to_ntc(src, dst, N, C, T, d_rs):
    _as(dst, (N * T, C), (d_rs, 1)).copy_(src[:N * C * T].view(N, C, T).permute(0, 2, 1)
                                           .reshape(N * T, C))


def pase_ntc_to_nct(src, s_rs, dst, N, C, T):
    v = _as(src, (N, T, C), (T * s_rs, s_rs, 1))
    dst[:N * C * T] = v.permute(0, 2, 1).reshape(-1)


def pase_qrnn_scan_fwd(Y, h, ldh, Cst, N, T, H):
    y = Y[:N * T * 3 * H].view(N, T, 3 * H)
    z, f, o = torch.tanh(y[..., :H]), torch.sigmoid(y[..., H:2 * H]), torch.sigmoid(y[..., 2 * H:])
    c = torch.zeros(N, H)
    cs = []
    for t in range(T):
        c = f[:, t] * z[:, t] + (1 - f[:, t]) * c
        cs.append(c)
    cst = torch.stack(cs, 1)
    Cst[:N * T * H] = cst.reshape(-1)
    _as(h, (N, T, H), (T * ldh, ldh, 1)).copy_(o * cst)


def pase_qrnn_scan_bwd(Y, Cst, dh, lddh, dY, N, T, H):
    y = Y[:N * T * 3 * H].view(N, T, 3 * H)
    z, f, o = torch.tanh(y[..., :H]), torch.sigmoid(y[..., H:2 * H]), torch.sigmoid(y[..., 2 * H:])
    c = Cst[:N * T * H].view(N, T, H)
    g = _as(dh, (N, T, H), (T * lddh, lddh, 1))
    out = torch.zeros(N, T, 3 * H)
    carry = torch.zeros(N, H)
    for t in range(T - 1, -1, -1):
        cm1 = c[:, t - 1] if t > 0 else torch.zeros(N, H)
        dc = g[:, t] * o[:, t] + carry
        out[:, t, :H] = dc * f[:, t] * (1 - z[:, t] ** 2)
        out[:, t, H:2 * H] = dc * (z[:, t] - cm1) * f[:, t] * (1 - f[:, t])
        out[:, t, 2 * H:] = g[:, t] * c[:, t] * o[:, t] * (1 - o[:, t])
        carry = dc * (1 - f[:, t])
    dY[:N * T * 3 * H] = out.reshape(-1)


def _ctx(label, B, F, T, r):
    lab = label[:B * F * T].view(B, F, T)
    pad = torch.nn.functional.pad(lab, (r // 2, r // 2))
    win = pad.unfold(2, r, 1)                                   # B,F,T,r
    return win.permute(0, 2, 1, 3).reshape(B * T, F * r)        # rows (b,t), cols f*r+j


def pase_ctx_mse_fwd(pred, ldp, label, B, F, T, r, acc):
    p = _as(pred, (B * T, F * r), (ldp, 1))
    acc[0] += ((p - _ctx(label, B, F, T, r)).double() ** 2).sum()


def pase_ctx_mse_bwd(pred, ldp, label, B, F, T, r, coef, gscale, dpred, lddp):
    p = _as(pred, (B * T, F * r), (ldp, 1))
    k = coef * (float(gscale[0]) if gscale is not None else 1.0)
    _as(dpred, (B * T, F * r), (lddp, 1)).copy_(k * (p - _ctx(label, B, F, T, r)))


def pase_l1_fwd(pred, target, n, acc):
    acc[0] += (pred[:n] - target[:n]).abs().double().sum()


def pase_l1_bwd(pred, target, n, coef, gscale, dpred):
    k = coef * (float(gscale[0]) if gscale is not None else 1.0)
    dpred[:n] = k * torch.sign(pred[:n] - target[:n])


def pase_bce_pairs_fwd(logit, n, n_pos, acc):
    # the kernel's stable element loss max(v, 0) - v y + log1p(e^-|v|) in fp32 (torch's
    # binary_cross_entropy_with_logits returns 0 for a confident y = 0 logit)
    v = logit[:n]
    y = (torch.arange(n) < n_pos).float()
    acc[0] += (v.clamp_min(0.0) - v * y + torch.log1p(torch.exp(-v.abs()))).double().sum()


def pase_bce_pairs_bwd(logit, n, n_pos, coef, gscale, dlogit):
    y = (torch.arange(n) < n_pos).float()
    k = coef * (float(gscale[0]) if gscale is not None else 1.0)
    dlogit[:n] = k * (torch.sigmoid(logit[:n]) - y)


def pase_time_mean_fwd(x, ldx, out, ldo, B, T, C):
    _as(out, (B, C), (ldo, 1)).copy_(_as(x, (B, T, C), (T * ldx, ldx, 1)).mean(1))


def pase_time_mean_bwd(dout, ldo, dx, ldx, B, T, C, accumulate):
    g = (_as(dout, (B, C), (ldo, 1)) / T)[:, None, :].expand(B, T, C)
    v = _as(dx, (B, T, C), (T * ldx, ldx, 1))
    if accumulate:
        v += g
    else:
        v.copy_(g)


def pase_axpy(x, y, n, a):
    y[:n] += a * x[:n]


def pase_scale_dev(x, n, dev_scalar, host_coef):
    x[:n] *= (float(dev_scalar[0]) if dev_scalar is not None else 1.0) * host_coef


def _host_view(ptr, n, dtype=torch.float32):
    """View of n elements at a HOST address (the emulation's stand-in for a device pointer
    stored in a job table); shares memory with the tensor that owns the address."""
    import ctypes
    import numpy as np
    if dtype == torch.float32:
        return torch.from_numpy(np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr)))
    raw = torch.from_numpy(np.ctypeslib.as_array((ctypes.c_int16 * n).from_address(ptr)))
    return raw.view(dtype)


def pase_conv_w_batch(table, njobs, total, op, dst_base, fmt):
    """ops 3..5: same results as 0..2 (shared-memory tiled kernels; `total` = thread blocks,
    table[.., 11] = first block of the job).  fmt: what hi/lo receive (0 tf32 split, 1 bf16,
    2 fp16 pair); dst may be 0."""
    t = table.reshape(njobs, 12).tolist()
    tiled, op = op >= 3, op % 3
    done = blocks = 0
    for (src, dst, hi, lo, Cout, Cin, k, sd, taps, start, count, bstart) in t:
        assert start == done
        if tiled:
            assert bstart == blocks and Cout % 32 == 0 and Cin % 8 == 0
            blocks += (Cout // 32) * (Cin // 8) if op == 1 else Cout
        n_w = Cout * Cin * k
        if op == 2:
            out = _host_view(dst_base.data_ptr() + 4 * dst, count)     # pointer arithmetic
            pase_conv_w_from_fwd(_host_view(src, n_w), out, Cout, Cin, k)
        else:
            out = _host_view(dst, count) if dst else torch.zeros(count)
            if op == 0:
                pase_conv_w_to_fwd(_host_view(src, n_w), out, Cout, Cin, k)
            else:
                pase_conv_w_to_dgrad(_host_view(src, n_w), out, Cout, Cin, k, sd, taps)
        if hi:
            if fmt == 0:
                pase_split_tf32(out, _host_view(hi, count), _host_view(lo, count), count)
            elif fmt == 1:
                _host_view(hi, count, torch.bfloat16).copy_(out.to(torch.bfloat16))
            else:
                pase_split_f16(out, _host_view(hi, count, torch.float16),
                               _host_view(lo, count, torch.float16), count, None, None)
        done += count
    assert (blocks if tiled else done) == total


# ---- tensor-core GEMM entry points (semantic spec: exact product of hi+lo operands) ----
def _tf32_trunc(x):
    return (x.contiguous().view(torch.int32) & -8192).view(torch.float32)


def _tf32_rn(x):
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    u = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    u = torch.where(u >= 2 ** 31, u - 2 ** 32, u)
    return u.to(torch.int32).view(torch.float32)


def pase_split_tf32(x, hi, lo, n):
    """hi None (activations): lo = rn(x - trunc(x)); hi given (weights): hi = rn(x),
    lo = rn(x - hi)."""
    if hi is not None:
        h = _tf32_rn(x[:n])
        hi[:n] = h
    else:
        h = _tf32_trunc(x[:n])
    lo[:n] = _tf32_rn(x[:n] - h)


def _like(lo, hi):
    """lo residual arrays may be shorter than the hi buffer (only the used part is split)."""
    if lo is None or lo.numel() >= hi.numel():
        return lo
    out = torch.zeros(hi.numel(), dtype=lo.dtype)
    out[:lo.numel()] = lo
    return out


def _operand(hi, lo, mode, n=None):
    """fp32 value of a GEMM operand as the tensor core sees it in `mode`."""
    hi = hi if n is None else hi[:n]
    if mode <= 1:
        v = _tf32_trunc(hi)
        if mode == 1:
            v = v + _tf32_trunc(lo if n is None else lo[:n])
        return v
    if mode == 2:
        assert hi.dtype == torch.bfloat16
        return hi.float()
    assert hi.dtype == torch.float16 and lo.dtype == torch.float16
    return hi.float() + (lo if n is None else lo[:n]).float() / F16_LO_MUL


def _tc_format(name, mode, Ahi, Alo, Bhi, Blo):
    """The mode checks both tensor-core entry points share (csrc/gemm_tc.cu), and the element
    type each mode reads; returns (element size, elements per 128-byte row)."""
    assert mode in (0, 1, 2, 3), "%s: mode %r" % (name, mode)
    assert mode not in (1, 3) or (Alo is not None and Blo is not None), \
        "%s: split modes need lo operands" % name
    dtype = (torch.float32, torch.float32, torch.bfloat16, torch.float16)[mode]
    for t in (Ahi, Alo, Bhi, Blo):
        assert t is None or t.dtype == dtype, "%s: mode %d operand dtype %s" % (name, mode, t.dtype)
    esz = dtype.itemsize
    return esz, 128 // esz


def pase_tc_gemm_nt(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, alpha, alpha_dev, bias,
                    rows_in, t_valid, rows_out, fold, colsum, colsumsq, accumulate, mode, c_bf16):
    # the PASE_CHECK_ARG preconditions of the C entry point: a shape it refuses fails here
    assert Ahi is not None and Bhi is not None and M > 0 and N > 0 and K > 0
    esz, eb = _tc_format("pase_tc_gemm_nt", mode, Ahi, Alo, Bhi, Blo)
    assert R >= eb and R % eb == 0, "pase_tc_gemm_nt: R=%d must be a multiple of %d" % (R, eb)
    assert (K * esz) % 16 == 0 and (ldb * esz) % 16 == 0 and ldb >= K, \
        "pase_tc_gemm_nt: K/ldb alignment (K=%d ldb=%d)" % (K, ldb)
    assert Ahi.data_ptr() % 16 == 0 and Bhi.data_ptr() % 16 == 0, \
        "pase_tc_gemm_nt: operand alignment"
    assert rows_in > 0 and rows_out > 0 and fold > 0 and N % fold == 0, \
        "pase_tc_gemm_nt: bad row map"
    assert (colsum is None) == (colsumsq is None) and (colsum is None or N <= 4096) and \
        (colsum is None or not accumulate), "pase_tc_gemm_nt: statistics"
    Alo, Blo = _like(Alo, Ahi), _like(Blo, Bhi)
    need = M * R + K
    A = torch.zeros(need)
    lim = min(a_rows * R, Ahi.numel(), need)         # TMA zero-fills rows >= a_rows
    A[:lim] = _operand(Ahi, Alo, mode, lim)
    B = _operand(Bhi, Blo, mode, N * ldb)
    if alpha_dev is not None:
        alpha = alpha * float(alpha_dev[0])
    if c_bf16:
        assert C.dtype == torch.bfloat16 and not accumulate
        Cf = C.float()
        pase_gemm_nt(A, R, B, ldb, Cf, ldc, M, N, K, alpha, bias, rows_in, t_valid, rows_out,
                     fold, colsum, colsumsq, 0)
        C.copy_(Cf.to(torch.bfloat16))
        return
    pase_gemm_nt(A, R, B, ldb, C, ldc, M, N, K, alpha, bias, rows_in, t_valid, rows_out, fold,
                 colsum, colsumsq, accumulate)


def pase_tc_gemm_tn(Ahi, Alo, lda, pitchA, offA, Bhi, Blo, R, pitchB, b_rows_total, C, ldc, I, J,
                    groups, rows_per_group, alpha, alpha_dev, accumulate, mode):
    assert Ahi is not None and Bhi is not None and I > 0 and J > 0 and groups > 0 and \
        rows_per_group > 0, "pase_tc_gemm_tn: bad args"
    esz, eb = _tc_format("pase_tc_gemm_tn", mode, Ahi, Alo, Bhi, Blo)
    assert R >= eb and R % eb == 0 and (lda * esz) % 16 == 0 and I % 4 == 0 and J % eb == 0, \
        "pase_tc_gemm_tn: need R%%%d==0, lda*%d%%16==0, I%%4==0, J%%%d==0 (R=%d lda=%d I=%d J=%d)" \
        % (eb, esz, eb, R, lda, I, J)
    Alo, Blo = _like(Alo, Ahi), _like(Blo, Bhi)
    A = _operand(Ahi, Alo, mode)
    needB = ((groups - 1) * pitchB + rows_per_group) * R + J
    B = torch.zeros(max(needB, Bhi.numel()))
    lim = min(b_rows_total * R, Bhi.numel())
    B[:lim] = _operand(Bhi, Blo, mode, lim)
    if alpha_dev is not None:
        alpha = alpha * float(alpha_dev[0])
    pase_gemm_tn(A, lda, pitchA, offA, B, R, pitchB, 0, C, ldc, I, J, groups, rows_per_group,
                 alpha, accumulate)


def pase_scatter_copy(table, njobs, total):
    t = table.reshape(njobs, 6).tolist()
    done = 0
    for (src, dst, rows, cols, sld, dld) in t:
        s = _host_view(src, (rows - 1) * sld + cols)
        d = _host_view(dst, (rows - 1) * dld + cols)
        _as(d, (rows, cols), (dld, 1)).copy_(_as(s, (rows, cols), (sld, 1)))
        done += rows * cols
    assert done == total


def pase_rownorm_max(X, ld, rows, cols, amax):
    v = _as(X, (rows, cols), (ld, 1)).double().pow(2).sum(1).sqrt().max()
    amax[0] = max(float(amax[0]), float(v))


def pase_bound_scale(a4, scale_out):
    s = f16_grad_scale((float(a4[0]) * float(a4[1]) + float(a4[2]) + float(a4[3])) * 1.0001)
    scale_out[0], scale_out[1] = 1.0 / s, s


def pase_frame_wave(x, N, T, hop, win, start0, frames, hi, lo, lda):
    idx = (torch.arange(frames)[:, None] * hop + start0 + torch.arange(win)[None, :])
    idx = _reflect(idx, T)
    A = torch.zeros(N, frames, lda)
    A[:, :, :win] = x[:N * T].view(N, T)[:, idx]
    h = A.to(torch.float16)
    hi[:N * frames * lda] = h.reshape(-1)
    lo[:N * frames * lda] = ((A - h.float()) * F16_LO_MUL).to(torch.float16).reshape(-1)


def pase_lps_post(C, ldc, N, frames, nbins, der_order, width, fir, mean, stdv, out):
    spec = _as(C, (N, frames, ldc), (frames * ldc, ldc, 1))
    re, im = spec[:, :, 0:2 * nbins:2], spec[:, :, 1:2 * nbins:2]
    mag = torch.sqrt(re * re + im * im)
    X = (10.0 * torch.log10(mag * mag + 1e-19)).permute(0, 2, 1)          # (N, nbins, frames)
    feats = [X]
    half = width // 2
    for d in range(1, der_order + 1):
        taps = fir[(d - 1) * width:d * width]
        c = torch.arange(frames).clamp(half, frames - 1 - half)
        win = c[:, None] - half + torch.arange(width)[None, :]               # (frames, width)
        feats.append((X[:, :, win] * taps).sum(-1))
    Y = torch.cat(feats, 1)
    if mean is not None:
        Y = (Y - mean[:Y.shape[1], None]) / stdv[:Y.shape[1], None]
    out[:Y.numel()] = Y.reshape(-1)
