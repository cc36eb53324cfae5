"""The loss side of the worker heads, one C-ABI entry point at a time: float64 references, the
error bounds the GPU tests hold the kernels to, and those bounds checked on the CPU emulation
(tests/emul/) at reduced shapes, so a wrong reference or bound shows before any GPU run.
tests/test_head_losses_gpu.py runs the same references and checks against the CUDA kernels at
the shapes the workers+ step runs them.

Entry points:
  pase_tc_gemm_nt_ctxmse   fused output layer of an MLP regression head: residual
                           d = h W^T + b - ctx_r(label) as a power-of-two scaled fp16 pair,
                           sum d^2 and the column sums of d (bias gradient); loss-only form;
  pase_ctx_mse_fwd/bwd     the unfused contextualised MSE on fp32 predictions;
  pase_bce_pairs_fwd/bwd   BCE-with-logits against the [ones; zeros] labels of LIM/GIM/SPC;
  pase_time_mean_fwd/bwd   GIM's mean over time.

Bounds (u = 2^-24), derived from the arithmetic of each kernel:
  fused residual   (rep + (D + 2) u) S + u |ctx(label)| + 2^-36 (sum_k |W_nk| + sum_k |h_mk|),
                   S = |h| |W|^T + |b| in float64: the 3xf16 GEMM bar of DESIGN.md section 5
                   (rep = 2^-20, D = 2 min(K, 512) + ceil(K / 128) + 128), one rounding for the
                   bias fmaf and one for the label subtraction, and 2^-36 per operand element
                   the fp16 pair holds below its normal range;
  residual pair    (Rhi + 2^-11 Rlo) / s within e + 2^-22 (|d| + e) + 2^-36 / s of d (fp16 hi and
                   lo' carry 11 bits each; lo' is subnormal-limited to 2^-36 of the scaled value);
  loss             sum (2 |d| e + e^2) + 64 u sum (|d| + e)^2: each consumer thread sums the
                   squares of its 64 elements of a 128-column tile with an fp32 fma chain, the
                   partials meet in fp64 (2^-40 of the magnitudes);
  column sums      sum_m e + 4 u sum_m (|d| + e): per 16-row group one fp32 add of a thread's two
                   rows and three shuffle adds, the groups meet in fp64;
  ctx-MSE fwd      (32 + 2) u sum d^2: the fp32 difference (2 u on d^2) and a 32-row fp32 fma
                   chain per thread (CTX_RPB), partials in fp64;
  ctx-MSE bwd      2 u |k (p - ctx(label))| with k = fp32(coef * g) as the kernel forms it (one
                   rounding for the difference, one for the product): within 2 ulp;
  BCE fwd          8 u per element (expf within 2 ulp, log1pf within 1 ulp, two adds) of the
                   float64 max(v, 0) - v y + log1p(e^-|v|), plus 2^-148 per element for the
                   subnormal e^-|v| of |v| > 87; below 1e-6 of the sum;
  BCE bwd          k (2 u sigma + 4 u sigma (1 - sigma) + 2 u |sigma - y|) + 2^-120 k: expf
                   within 2 ulp, the 1 + t add and the division, the subtraction of y (exact but
                   for y = 1, sigma < 1/2) and the product with k; the floor covers e^-v
                   overflowing (sigma < 2^-126 read as 0).  k = fp32(coef * g) as the kernel
                   forms it;
  time mean fwd    T u sum_t |x| / T (a sequential fp32 sum over T, then one division);
  time mean bwd    exact: fp32(dout / T), added to the old dx in fp32 when accumulating."""
import math

import pytest
import torch

import emul
import pase_b200.ops as ops
from pase_b200 import gemm
from pase_oracle import contextualize, _CRIT
from test_decoder_gpu import _within, _report

U = 2.0 ** -24
F16X3 = gemm.PRECISIONS["3xf16"]
REP_F16X3 = 2.0 ** -20       # representation error of a 3xf16 product (DESIGN.md section 5)
CTX_RPB = 32                 # rows one thread of pase_ctx_mse_* sums (csrc/loss.cu)
D2_DEPTH = 64                # squares one consumer thread of the fused epilogue sums per tile
DB_DEPTH = 4                 # fp32 adds of a column sum over one 16-row group
F64_SUM = 2.0 ** -40         # fp64 combination of the partials, relative to the magnitudes
F16_SENTINEL = 1234.0        # rows past M of the residual pair keep this


def _f64(x):
    return torch.tensor([x], dtype=torch.float64)


def ldr_of(N):
    return -(-N // 128) * 128


def split_depth(K):
    return 2 * min(K, 512) + -(-K // 128) + 128


def f16_scale64(bound):
    """The power of two s with bound * 1.0001 * s <= 2^14, in float64 (f16_grad_scale)."""
    bound = bound * 1.0001
    if not (0.0 < bound < 3.0e38):
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, 14 - math.frexp(bound)[1])))


# ---- float64 references ----
def ctx64(label, r, m0=0, m1=None):
    """Rows [m0, m1) of ctx_r(label) in float64: row m = (b, t) = divmod(m, T), column f r + j
    holds label[b, f, t + j - r // 2], zero outside [0, T)."""
    B, F, T = label.shape
    m1 = B * T if m1 is None else m1
    m = torch.arange(m0, m1, device=label.device)
    b, t = m // T, m % T
    tt = t[:, None] + torch.arange(r, device=label.device)[None, :] - r // 2     # (rows, r)
    ok = (tt >= 0) & (tt < T)
    v = label.double()[b[:, None], :, tt.clamp(0, T - 1)]                        # (rows, r, F)
    v = torch.where(ok[:, :, None], v, torch.zeros_like(v))
    return v.permute(0, 2, 1).reshape(m1 - m0, F * r)


def residual64(h, W, b, label, r, m0, m1):
    """Rows [m0, m1) of d = h W^T + b - ctx_r(label) in float64, the matching S = |h| |W|^T + |b|
    and |ctx_r(label)|."""
    h64, W64 = h[m0:m1].double(), W.double()
    lab = ctx64(label, r, m0, m1)
    d = h64 @ W64.t() - lab
    S = h64.abs() @ W64.abs().t()
    if b is not None:
        d += b.double()[None, :]
        S += b.double().abs()[None, :]
    return d, S, lab.abs()


def residual_bound(S, lab_abs, K, ha_sum, wa_sum):
    """Per-element bound of the fused kernel's fp32 residual; ha_sum (rows, 1) = sum_k |h_mk|,
    wa_sum (1, N) = sum_k |W_nk|."""
    return (REP_F16X3 + (split_depth(K) + 2) * U) * S + U * lab_abs + \
        2.0 ** -36 * (ha_sum + wa_sum)


def pair_bound(d, e, s):
    return e + 2.0 ** -22 * (d.abs() + e) + 2.0 ** -36 / s


def loss_bound_terms(d, e):
    """This block's share of the loss bound."""
    m2 = (d.abs() + e) ** 2
    return float((2 * d.abs() * e + e * e).sum() + (D2_DEPTH * U + F64_SUM) * m2.sum())


def db_bound_terms(d, e):
    return e.sum(0) + (DB_DEPTH * U + F64_SUM) * (d.abs() + e).sum(0)


def ctx_mse_ref(pred, ldp, label, r):
    """sum (p - ctx_r(label))^2 in float64 and its bound."""
    B, F, T = label.shape
    N = F * r
    p = pred.view(-1, ldp)[:B * T, :N].double()
    d2 = ((p - ctx64(label, r)) ** 2).sum()
    return float(d2), float((CTX_RPB + 2) * U * d2 + F64_SUM * d2)


def ctx_mse_grad_ref(pred, ldp, label, r, coef, g):
    """k (p - ctx_r(label)) in float64 with k = fp32(coef * g), and its bound."""
    B, F, T = label.shape
    N = F * r
    k = torch.tensor(coef, dtype=torch.float32)
    if g is not None:
        k = k * g.cpu().float()[0]
    p = pred.view(-1, ldp)[:B * T, :N].double()
    ref = float(k) * (p - ctx64(label, r))
    return ref, 2 * U * (1 + U) * ref.abs()


def bce_ref(logit, n_pos):
    """sum_i max(v, 0) - v y + log1p(e^-|v|) in float64 (y = 1 for i < n_pos) and its bound."""
    v = logit.double()
    y = (torch.arange(v.numel(), device=v.device) < n_pos).double()
    el = v.clamp_min(0.0) - v * y + torch.log1p(torch.exp(-v.abs()))
    return float(el.sum()), float(8 * U * el.abs().sum()) + v.numel() * 2.0 ** -148


def bce_grad_ref(logit, n_pos, coef, g):
    """k (sigma(v) - y) in float64 with k = fp32(coef * g), and its bound."""
    k = torch.tensor(coef, dtype=torch.float32)
    if g is not None:
        k = k * g.cpu().float()[0]
    k = float(k)
    v = logit.double()
    y = (torch.arange(v.numel(), device=v.device) < n_pos).double()
    sg = torch.sigmoid(v)
    tol = k * (2 * U * sg + 4 * U * sg * (1 - sg) + 2 * U * (sg - y).abs()) * (1 + 2.0 ** -20) \
        + k * 2.0 ** -120
    return k * (sg - y), tol


def time_mean_ref(x, ldx, B, T, C):
    v = x.view(-1, ldx)[:B * T, :C].double().view(B, T, C)
    return v.mean(1), U * v.abs().sum(1)


# ---- the fused regression head, operands through the product's own path ----
def run_fused(h, W, b, label, r, loss_only=False, extra_rows=3):
    """pase_tc_gemm_nt_ctxmse as _FusedLinearCtxMSE.forward launches it (gemm.to_operand for h
    and W, the Cauchy-Schwarz scale chain), the pair allocated with `extra_rows` sentinel rows
    past M.  -> dict of the kernel's outputs."""
    rows, K = h.shape
    N = W.shape[0]
    B, F, T = label.shape
    dev = h.device
    ldr = ldr_of(N)
    hop = gemm.to_operand(F16X3, h.reshape(-1), rows * K)
    wop = gemm.to_operand(F16X3, W.reshape(-1), N * K, "weight")
    if loss_only:
        acc = torch.zeros(1, dtype=torch.float64, device=dev)
        ops.call("pase_tc_gemm_nt_ctxmse", hop.hi, hop.lo, rows, K, wop.hi, wop.lo, K, None,
                 None, ldr, rows, N, K, b, label.reshape(-1), B, F, T, r, None, acc, None)
        return {"loss": float(acc[0])}
    am = torch.zeros(4, dtype=torch.float32, device=dev)
    ops.call("pase_rownorm_max", h.reshape(-1), K, rows, K, am[0:1])
    ops.call("pase_rownorm_max", W.reshape(-1), K, N, K, am[1:2])
    if b is not None:
        ops.call("pase_absmax", b, N, am[2:3])
    ops.call("pase_absmax", label.reshape(-1), label.numel(), am[3:4])
    scale = torch.empty(2, dtype=torch.float32, device=dev)
    ops.call("pase_bound_scale", am, scale)
    n_pair = (rows + extra_rows) * ldr
    Rhi = torch.full((n_pair,), F16_SENTINEL, dtype=torch.float16, device=dev)
    Rlo = torch.full((n_pair,), F16_SENTINEL, dtype=torch.float16, device=dev)
    acc = torch.zeros(1 + ldr, dtype=torch.float64, device=dev)
    ops.call("pase_tc_gemm_nt_ctxmse", hop.hi, hop.lo, rows, K, wop.hi, wop.lo, K, Rhi, Rlo, ldr,
             rows, N, K, b, label.reshape(-1), B, F, T, r, scale, acc[0:1], acc[1:])
    return {"loss": float(acc[0]), "db": acc[1:], "Rhi": Rhi.view(-1, ldr),
            "Rlo": Rlo.view(-1, ldr), "scale": scale.tolist(), "ldr": ldr}


def check_fused(h, W, b, label, r, out, chunk=1024, loss_only=None):
    """Every output of one run_fused call against float64 from the kernel's inputs.
    loss_only: the loss of the loss-only form, held to the same bound.  -> {what: worst
    err / bound} and the floor 2^-36 / s over rms(d)."""
    rows, K = h.shape
    N = W.shape[0]
    ldr = out["ldr"]
    inv_s, s = out["scale"]
    ratios = {}
    # the scale: the power of two from the four maxima, recomputed in float64
    bound = float(h.double().norm(dim=1).max()) * float(W.double().norm(dim=1).max()) + \
        float(label.double().abs().max())
    if b is not None:
        bound += float(b.double().abs().max())
    assert s == f16_scale64(bound) and inv_s == 1.0 / s, (out["scale"], bound)
    Rhi, Rlo = out["Rhi"], out["Rlo"]
    assert bool((Rhi[rows:] == F16_SENTINEL).all()) and bool((Rlo[rows:] == F16_SENTINEL).all()), \
        "residual pair: rows past M written"
    assert bool((Rhi[:rows, N:] == 0).all()) and bool((Rlo[:rows, N:] == 0).all()), \
        "residual pair: columns [N, ldr) not zero"
    assert float(Rhi[:rows].float().abs().max()) <= 2.0 ** 14, "residual pair: |Rhi| > 2^14"
    assert bool((out["db"][N:] == 0).all()), "db_acc: columns past N written"
    wa_sum = W.double().abs().sum(1)[None, :]
    loss_ref = loss_tol = sum_d2 = 0.0
    db_ref = torch.zeros(N, dtype=torch.float64, device=h.device)
    db_tol = torch.zeros_like(db_ref)
    for m0 in range(0, rows, chunk):
        m1 = min(rows, m0 + chunk)
        d, S, lab_abs = residual64(h, W, b, label, r, m0, m1)
        e = residual_bound(S, lab_abs, K, h[m0:m1].double().abs().sum(1, keepdim=True), wa_sum)
        del S, lab_abs
        v = (Rhi[m0:m1, :N].double() + Rlo[m0:m1, :N].double() / 2048.0) * inv_s
        ratios["pair"] = max(ratios.get("pair", 0.0), _within("pair", v, d, pair_bound(d, e, s)))
        del v
        loss_ref += float((d * d).sum())
        sum_d2 += float((d * d).sum())
        loss_tol += loss_bound_terms(d, e)
        db_ref += d.sum(0)
        db_tol += db_bound_terms(d, e)
        del d, e
    ratios["loss"] = _within("loss", _f64(out["loss"]), _f64(loss_ref), loss_tol)
    if loss_only is not None:
        ratios["loss_only"] = _within("loss-only", _f64(loss_only), _f64(loss_ref), loss_tol)
    ratios["db"] = _within("db", out["db"][:N], db_ref, db_tol)
    floor = 2.0 ** -36 / s / math.sqrt(sum_d2 / (rows * N))
    return ratios, floor


def init_head(B, T, F, r, K, dev, seed=0, bias=True):
    """Operands at their initial scale: post-PReLU-like h ~ N(0, 1), W ~ N(0, 1 / K) (the
    nn.Linear init variance order), b ~ 0.1 N(0, 1), label ~ N(0, 1), all fp32."""
    gen = torch.Generator().manual_seed(7000 + seed)
    N = F * r
    h = torch.randn(B * T, K, generator=gen)
    W = torch.randn(N, K, generator=gen) / math.sqrt(K)
    b = 0.1 * torch.randn(N, generator=gen) if bias else None
    label = torch.randn(B, F, T, generator=gen)
    return [t if t is None else t.to(dev) for t in (h, W, b, label)]


def fitted_head(B, T, F, K, dev, seed=0):
    """A head that has fitted its target (r = 1): label = h W^T + b + noise at 1e-3 of the
    label's scale, so |d| is ~1e-3 of the Cauchy-Schwarz bound that sets s."""
    h, W, b, _ = init_head(B, T, F, 1, K, "cpu", seed)
    gen = torch.Generator().manual_seed(7500 + seed)
    y = (h.double() @ W.double().t() + b.double()).view(B, T, F)
    y = y + 1e-3 * y.std() * torch.randn(y.shape, generator=gen, dtype=torch.float64)
    label = y.permute(0, 2, 1).contiguous().float()
    return [t.to(dev) for t in (h, W, b, label)]


def loose_head(B, T, F, r, K, dev, seed=0, n_big=5):
    """A loose scale: n_big rows of h with 100x the typical norm set s; the other rows'
    residuals sit far below the bound."""
    h, W, b, label = init_head(B, T, F, r, K, "cpu", seed)
    gen = torch.Generator().manual_seed(7700 + seed)
    idx = torch.randperm(B * T, generator=gen)[:n_big]
    h[idx] *= 100.0
    return [t.to(dev) for t in (h, W, b, label)]


# ---- on the CPU emulation ----
@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)


EMUL_FUSED = {                    # (B, T, F, r, K, bias)
    "one-tile": (3, 50, 11, 7, 128, True),
    "n-tail": (2, 70, 20, 7, 64, True),            # N = 140: a second, partial column tile
    "short-T": (5, 2, 9, 7, 64, True),
    "flush-kb": (2, 40, 5, 3, 576, False),
}


@pytest.mark.parametrize("case", list(EMUL_FUSED))
def test_fused_emulated_within_bounds(emulated, case):
    B, T, F, r, K, bias = EMUL_FUSED[case]
    h, W, b, label = init_head(B, T, F, r, K, "cpu", seed=len(case), bias=bias)
    out = run_fused(h, W, b, label, r)
    only = run_fused(h, W, b, label, r, loss_only=True)["loss"]
    ratios, floor = check_fused(h, W, b, label, r, out, chunk=64, loss_only=only)
    _report("fused emulated " + case, ratios.items())
    assert floor < 1e-6


@pytest.mark.parametrize("regime", ["fitted", "loose"])
def test_fused_emulated_regimes(emulated, regime):
    if regime == "fitted":
        h, W, b, label = fitted_head(2, 60, 130, 64, "cpu")
        r = 1
    else:
        h, W, b, label = loose_head(2, 60, 20, 7, 64, "cpu")
        r = 7
    ratios, floor = check_fused(h, W, b, label, r, run_fused(h, W, b, label, r))
    _report("fused emulated " + regime, ratios.items())
    assert floor < 1e-6, "2^-36 / s is %.3g of rms(d)" % floor


def test_ctx64_matches_oracle_and_loss():
    """ctx64 against pase_oracle.contextualize, and the fused reference's mean of d^2 against
    the oracle's MSE of the (B, F r, T) prediction."""
    B, T, F, r, K = 3, 9, 4, 7, 64
    h, W, b, label = init_head(B, T, F, r, K, "cpu", seed=3)
    ref = contextualize(label.double(), r)                       # (B, F r, T)
    assert torch.equal(ctx64(label, r), ref.permute(0, 2, 1).reshape(B * T, F * r))
    for rr in (1, 3):
        assert torch.equal(ctx64(label, rr),
                           contextualize(label.double(), rr).permute(0, 2, 1).reshape(B * T, -1))
    d, _, _ = residual64(h, W, b, label, r, 0, B * T)
    pred = (h.double() @ W.double().t() + b.double()).view(B, T, F * r).permute(0, 2, 1)
    mse = _CRIT["MSELoss"](pred, ref)
    assert abs(float((d * d).mean()) - float(mse)) <= 1e-12 * float(mse)


@pytest.mark.parametrize("B,T,F,r", [(2, 21, 13, 7), (3, 1, 5, 3), (2, 33, 40, 7), (4, 2, 6, 1)])
def test_ctx_mse_emulated_within_bounds(B, T, F, r):
    gen = torch.Generator().manual_seed(B * T + r)
    ldp = F * r + 5
    pred = torch.randn(B * T * ldp, generator=gen)
    label = torch.randn(B, F, T, generator=gen)
    acc = torch.zeros(1, dtype=torch.float64)
    emul.call("pase_ctx_mse_fwd", pred, ldp, label.reshape(-1), B, F, T, r, acc)
    ref, tol = ctx_mse_ref(pred, ldp, label, r)
    _within("ctx_mse_fwd", acc, _f64(ref), tol)
    g = torch.tensor([0.7])
    dpred = torch.full((B * T * ldp,), 5.0)
    emul.call("pase_ctx_mse_bwd", pred, ldp, label.reshape(-1), B, F, T, r, 0.01, g, dpred, ldp)
    ref, tol = ctx_mse_grad_ref(pred, ldp, label, r, 0.01, g)
    _within("ctx_mse_bwd", dpred.view(-1, ldp)[:, :F * r], ref, tol)
    assert bool((dpred.view(-1, ldp)[:, F * r:] == 5.0).all())


def confident_logits(n, n_pos, seed=0, lo=17.0, hi=100.0):
    """Every pair classified confidently correctly: v in [lo, hi] for y = 1, in [-hi, -lo]
    for y = 0."""
    gen = torch.Generator().manual_seed(8000 + seed)
    v = lo + (hi - lo) * torch.rand(n, generator=gen)
    v[n_pos:] = -v[n_pos:]
    return v


def spread_logits(n, seed=0):
    """|v| uniform in [0, 100], random sign."""
    gen = torch.Generator().manual_seed(8100 + seed)
    v = 100.0 * torch.rand(n, generator=gen)
    return torch.where(torch.rand(n, generator=gen) < 0.5, -v, v)


@pytest.mark.parametrize("kind", ["confident", "spread", "edges"])
def test_bce_emulated_matches_float64(kind):
    """The emulated forward equals float64 to its bound, including a batch whose pairs are
    all confidently correct (its loss is ~1e-8 per pair, not 0)."""
    n, n_pos = 64, 32
    if kind == "confident":
        v = confident_logits(n, n_pos)
    elif kind == "spread":
        v = spread_logits(n)
    else:
        v = torch.tensor([18.0, 25.0, 40.0, 90.0, -18.0, -25.0, -40.0, -90.0])
        n, n_pos = 8, 4
    acc = torch.zeros(1, dtype=torch.float64)
    emul.call("pase_bce_pairs_fwd", v, n, n_pos, acc)
    ref, tol = bce_ref(v, n_pos)
    assert ref > 0.0
    assert tol <= 1e-6 * ref
    _within("bce_fwd", acc, _f64(ref), tol)
    d = torch.zeros(n)
    g = torch.tensor([0.75])
    emul.call("pase_bce_pairs_bwd", v, n, n_pos, 1.0 / 64, g, d)
    ref, tol = bce_grad_ref(v, n_pos, 1.0 / 64, g)
    _within("bce_bwd", d, ref, tol)


def test_time_mean_emulated():
    B, T, C, ldx, ldo = 3, 17, 40, 48, 44
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(B * T * ldx, generator=gen)
    out = torch.full((B * ldo,), 9.0)
    emul.call("pase_time_mean_fwd", x, ldx, out, ldo, B, T, C)
    ref, tol = time_mean_ref(x, ldx, B, T, C)
    _within("time_mean_fwd", out.view(B, ldo)[:, :C], ref, tol)
    assert bool((out.view(B, ldo)[:, C:] == 9.0).all())
