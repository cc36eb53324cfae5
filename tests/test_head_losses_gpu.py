"""The worker heads' loss kernels on the device against float64 computed with torch on the same
device from each kernel's own fp32 inputs, at the shapes the workers+ step runs them (B = 32,
T' = 200, K = 256; lps also at B = 64, T' = 300) and at their edges.  References, bounds and
their derivation: tests/test_head_losses.py.  Each test prints its worst element as a fraction
of its bound."""
import pytest
import torch

from pase_b200 import _lib
from pase_b200 import functional as Fn
from test_decoder_gpu import _within, _report
from test_head_losses import (
    U, REP_F16X3, split_depth, f16_scale64, ctx64, residual_bound, pair_bound, loss_bound_terms,
    db_bound_terms, ctx_mse_ref, ctx_mse_grad_ref, bce_ref, bce_grad_ref, time_mean_ref,
    run_fused, check_fused, init_head, fitted_head, loose_head, confident_logits, spread_logits,
    ldr_of, _f64)

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL = 2.0 ** 100

# workers+ regression heads: name -> F (num_outputs); r = 7 and K = 256 for all
WORKERS = {"lps": 3075, "fbank": 120, "mfcc": 39, "mfcc_long": 60, "prosody": 12}


def _fused(h, W, b, label, r, name):
    out = run_fused(h, W, b, label, r)
    only = run_fused(h, W, b, label, r, loss_only=True)["loss"]
    torch.cuda.synchronize()
    ratios, floor = check_fused(h, W, b, label, r, out, loss_only=only)
    _report(name, ratios.items())
    return floor


# ---- 1. the fused regression head at the workers+ shapes ----
@pytest.mark.parametrize("B,T,worker", [(32, 200, w) for w in WORKERS] + [(64, 300, "lps")])
def test_fused_ctxmse_workers_shapes(B, T, worker):
    h, W, b, label = init_head(B, T, WORKERS[worker], 7, 256, DEV, seed=B + len(worker))
    _fused(h, W, b, label, 7, "fused %s B=%d T=%d" % (worker, B, T))


# ---- 2. its edges ----
FUSED_EDGES = {                   # (B, T, F, r, K, bias)
    "T=1": (6, 1, 40, 7, 256, True),
    "T=2": (6, 2, 40, 7, 256, True),
    "T=3": (6, 3, 40, 7, 256, True),
    "B*T=185": (5, 37, 120, 7, 256, True),
    "r=1": (8, 50, 60, 1, 256, True),
    "r=3": (8, 50, 12, 3, 256, True),
    "K=64": (8, 50, 39, 7, 64, True),
    "K=576": (4, 100, 120, 7, 576, True),
    "K=1024": (4, 100, 120, 7, 1024, True),
    "no-bias": (5, 37, 39, 7, 256, False),
}


@pytest.mark.parametrize("case", list(FUSED_EDGES))
def test_fused_ctxmse_edges(case):
    B, T, F, r, K, bias = FUSED_EDGES[case]
    h, W, b, label = init_head(B, T, F, r, K, DEV, seed=7 * B + T, bias=bias)
    _fused(h, W, b, label, r, "fused " + case)


# ---- 3. magnitude regimes: the floor 2^-36 / s against the residual's own scale ----
@pytest.mark.parametrize("regime", ["init", "fitted", "loose"])
def test_fused_ctxmse_regimes(regime):
    B, T, K = 8, 200, 256
    if regime == "init":
        h, W, b, label = init_head(B, T, 120, 7, K, DEV, seed=11)
        r = 7
    elif regime == "fitted":
        h, W, b, label = fitted_head(B, T, 1025, K, DEV, seed=12)
        r = 1
    else:
        h, W, b, label = loose_head(B, T, 120, 7, K, DEV, seed=13)
        r = 7
    floor = _fused(h, W, b, label, r, "fused regime " + regime)
    print("fused regime %s: 2^-36 / s = %.3g rms(d)" % (regime, floor))
    assert floor < 1e-6, "regime %s: the pair's floor 2^-36 / s is %.3g of rms(d)" % (regime,
                                                                                      floor)


# ---- 4. the fused head's backward as the step runs it ----
def test_fused_head_backward_lps():
    """Fn.fused_linear_ctx_mse forward and backward at the lps shape: dh, dW and db against
    float64 autograd on the same fp32 h, W, b and label.  dh and dW are 3xf16 GEMMs whose
    residual operand is the fp16 pair: their bound is the GEMM bar with S taken over
    |d| + eps (eps the pair's bound), plus sum eps |other operand|, 2^-36 per element of the
    unscaled operand (h or W) below the fp16 normal range, and 4 u S for the device scalar
    g coef / s and the output rounding.  db: coef g times the column-sum bound, plus three
    roundings (fp64 -> fp32 with coef, times g)."""
    B, T, F, r, K = 32, 200, WORKERS["lps"], 7, 256
    h, W, b, label = init_head(B, T, F, r, K, DEV, seed=21)
    rows, N = B * T, F * r
    g = 0.75
    hp = h.clone().requires_grad_(True)
    Wp = torch.nn.Parameter(W.clone())
    bp = torch.nn.Parameter(b.clone())
    loss = Fn.fused_linear_ctx_mse(hp, Wp, bp, label, F, r)
    loss.backward(torch.tensor(g, device=DEV))
    torch.cuda.synchronize()
    # float64 autograd from the same fp32 values
    h64 = h.double().requires_grad_(True)
    W64 = W.double().requires_grad_(True)
    b64 = b.double().requires_grad_(True)
    d64 = h64 @ W64.t() + b64 - ctx64(label, r)
    l64 = (d64 * d64).mean()
    l64.backward(torch.tensor(g, dtype=torch.float64, device=DEV))
    with torch.no_grad():
        d = d64.detach()
        del d64
        # the fp32 residual's bound and the pair's, with s from the four maxima
        S = h.double().abs() @ W.double().abs().t() + b.double().abs()
        e = residual_bound(S, ctx64(label, r).abs(), K, h.double().abs().sum(1, keepdim=True),
                           W.double().abs().sum(1)[None, :])
        del S
        s = f16_scale64(float(h.double().norm(dim=1).max()) * float(W.double().norm(dim=1).max())
                        + float(b.double().abs().max()) + float(label.double().abs().max()))
        eps = pair_bound(d, e, s)
        # the loss: sum d^2 / (rows N), rounded to fp32
        tol = loss_bound_terms(d, e) / (rows * N) + U * float(l64)
        ratios = [("loss", _within("loss", _f64(float(loss)), _f64(float(l64)), tol))]
        cg = g * 2.0 / (rows * N)
        da = d.abs() + eps
        # dh = cg d W: the reduction runs over the ldr columns of the pair
        Wa = W.double().abs()
        Sh = da @ Wa
        tol_h = cg * ((REP_F16X3 + (split_depth(ldr_of(N)) + 4) * U) * Sh + eps @ Wa +
                      2.0 ** -36 * d.abs().sum(1, keepdim=True))
        ratios.append(("dh", _within("dh", hp.grad, h64.grad, tol_h)))
        del Sh, tol_h, Wa
        # dW = cg d^T h: the reduction runs over the rows
        Ha = h.double().abs()
        Sw = da.t() @ Ha
        tol_w = cg * ((REP_F16X3 + (split_depth(rows) + 4) * U) * Sw + eps.t() @ Ha +
                      2.0 ** -36 * d.abs().sum(0)[:, None])
        ratios.append(("dW", _within("dW", Wp.grad, W64.grad, tol_w)))
        del Sw, tol_w, Ha
        tol_b = cg * db_bound_terms(d, e) + 3 * U * b64.grad.abs()
        ratios.append(("db", _within("db", bp.grad, b64.grad, tol_b)))
    _report("fused backward lps", ratios)


# ---- 5. the unfused contextualised MSE ----
CTX_CASES = {                     # (B, T, F, r, ldp extra)
    "lps B=32": (32, 200, 3075, 7, 11),
    "lps B=64 T=300": (64, 300, 3075, 7, 3),
    "T=1 r=7": (9, 1, 40, 7, 5),
    "T=2 r=3": (9, 2, 40, 3, 5),
    "T=3 r=7": (9, 3, 40, 7, 5),
    "T=33 r=1": (7, 33, 300, 1, 5),
    "T=33 r=7": (7, 33, 39, 7, 1),
}


@pytest.mark.parametrize("case", list(CTX_CASES))
def test_ctx_mse(case):
    """T' = 200 and 33 are not multiples of CTX_RPB, so row blocks cross utterances; the
    columns [F r, ldp) of dpred keep their sentinel."""
    B, T, F, r, extra = CTX_CASES[case]
    N = F * r
    ldp = N + extra
    gen = torch.Generator(device=DEV).manual_seed(B * T + F)
    pred = torch.randn(B * T * ldp, device=DEV, generator=gen)
    label = torch.randn(B, F, T, device=DEV, generator=gen)
    acc = torch.zeros(1, dtype=torch.float64, device=DEV)
    _lib.call("pase_ctx_mse_fwd", pred, ldp, label.reshape(-1), B, F, T, r, acc)
    dpred = torch.full((B * T * ldp,), SENTINEL, device=DEV)
    coef = 2.0 / (B * T * N)
    gs = torch.tensor([0.75], device=DEV)
    _lib.call("pase_ctx_mse_bwd", pred, ldp, label.reshape(-1), B, F, T, r, coef, gs, dpred, ldp)
    torch.cuda.synchronize()
    ref, tol = ctx_mse_ref(pred, ldp, label, r)
    ratios = [("fwd", _within("ctx_mse_fwd", acc, _f64(ref).to(DEV), tol))]
    ref, tol = ctx_mse_grad_ref(pred, ldp, label, r, coef, gs)
    dv = dpred.view(-1, ldp)
    ratios.append(("bwd", _within("ctx_mse_bwd", dv[:, :N], ref, tol)))
    assert bool((dv[:, N:] == SENTINEL).all()), "ctx_mse_bwd wrote a padding column"
    _report("ctx_mse " + case, ratios)


# ---- 6. BCE against the pair labels ----
BCE_CASES = {                     # (n, logits)
    "lim B=32 spread": (64, "spread"),
    "grid-stride spread": (10 ** 6, "spread"),
    "lim B=32 confident": (64, "confident"),
    "grid-stride confident": (10 ** 6, "confident"),
}


@pytest.mark.parametrize("case", list(BCE_CASES))
def test_bce_pairs(case):
    """The forward's sum within 8 u of the element magnitudes of float64 (below 1e-6 of the
    sum), a batch of confidently correct pairs included; the backward elementwise."""
    n, kind = BCE_CASES[case]
    n_pos = n // 2
    v = (confident_logits(n, n_pos, seed=n) if kind == "confident" else spread_logits(n, seed=n))
    v = v.to(DEV)
    acc = torch.zeros(1, dtype=torch.float64, device=DEV)
    _lib.call("pase_bce_pairs_fwd", v, n, n_pos, acc)
    coef = 1.0 / n
    gs = torch.tensor([0.75], device=DEV)
    d = torch.full((n,), SENTINEL, device=DEV)
    _lib.call("pase_bce_pairs_bwd", v, n, n_pos, coef, gs, d)
    d1 = torch.full((n,), SENTINEL, device=DEV)
    _lib.call("pase_bce_pairs_bwd", v, n, n_pos, coef, None, d1)
    torch.cuda.synchronize()
    ref, tol = bce_ref(v, n_pos)
    assert tol <= 1e-6 * ref
    ratios = [("fwd", _within("bce_fwd", acc, _f64(ref).to(DEV), tol))]
    ref, tol = bce_grad_ref(v, n_pos, coef, gs)
    ratios.append(("bwd", _within("bce_bwd", d, ref, tol)))
    ref, tol = bce_grad_ref(v, n_pos, coef, None)
    ratios.append(("bwd g=None", _within("bce_bwd", d1, ref, tol)))
    _report("bce_pairs " + case, ratios)


# ---- 7. GIM's time mean ----
@pytest.mark.parametrize("accumulate", [0, 1])
def test_time_mean_gim(accumulate):
    B, T, C, ldx, ldo = 32, 200, 256, 320, 264
    gen = torch.Generator(device=DEV).manual_seed(31 + accumulate)
    x = torch.randn(B * T * ldx, device=DEV, generator=gen)
    out = torch.full((B * ldo,), SENTINEL, device=DEV)
    _lib.call("pase_time_mean_fwd", x, ldx, out, ldo, B, T, C)
    dout = torch.randn(B * ldo, device=DEV, generator=gen)
    dx = torch.randn(B * T * ldx, device=DEV, generator=gen)
    old = dx.clone()
    _lib.call("pase_time_mean_bwd", dout, ldo, dx, ldx, B, T, C, accumulate)
    torch.cuda.synchronize()
    ref, tol = time_mean_ref(x, ldx, B, T, C)
    ov = out.view(B, ldo)
    ratios = [("fwd", _within("time_mean_fwd", ov[:, :C], ref, tol))]
    assert bool((ov[:, C:] == SENTINEL).all()), "time_mean_fwd wrote past C"
    gref = (dout.view(B, ldo)[:, :C].cpu() / float(T))[:, None, :].expand(B, T, C)
    ov, dv = old.view(B, T, ldx).cpu(), dx.view(B, T, ldx).cpu()
    exp = ov[:, :, :C] + gref if accumulate else gref
    assert torch.equal(dv[:, :, :C], exp), "time_mean_bwd is not fp32(dout / T) exactly"
    assert torch.equal(dv[:, :, C:], ov[:, :, C:]), "time_mean_bwd wrote past C"
    _report("time_mean accumulate=%d" % accumulate, ratios)
