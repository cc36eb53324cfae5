"""The cchunk waveform decoder (DecoderMinion, pase_b200/decoder.py) against a float64 reference
computed with torch on the device from the same fp32 inputs, at the workers+ geometry the
training step runs (B = 32, T' = 200: 256 -> 512 -> 256 -> 128 channels, k = 30, strides
4 / 4 / 10, L = 32000) in every GEMM precision, and at the geometry edges of _LayerGeom.

Each stage is checked from the kernel's own input to that stage (the plan's buffers xz, yfull,
dyfull, dx), so errors and PReLU gate flips do not compound:
  forward GEMM   yfull[i] from xz[i], W and the bias repeated over the s phases;
  crop + PReLU   xz[i+1] (or the output) from yfull[i]: exact (one fp32 product);
  du             dyfull[i] inside each sample's crop window from yfull[i] and the incoming
                 gradient: exact; outside the window exactly 0 (the GEMMs read it);
  db, dalpha     fp64 sums over B*L positions;
  dW             from dyfull[i] and xz[i] (every sample);
  dx             dx[i] from dyfull[i] and W;
  3xf16          the gradient operand of dyfull[i] (hi + 2^-11 lo') / s within
                 2^-22 |dy| + 2^-36 / s of dy, with s the power of two f16_grad_scale gives.
The float64 reference of the polyphase GEMMs is built from W by index arithmetic (poly_weight,
fwd_gemm_checks, bwd_checks); tests/test_decoder_emulated.py runs the same checks on the CPU
emulation and checks the emulated decoder against torch's conv_transpose1d.

Bounds (u = 2^-24).  For a GEMM output with K products, S = the same operation on |A| and |B|
(+ |bias|) in float64, the error is at most (rep + D u) S + floor:
  D     accumulation depth, at most 2 u per add in the tensor core's own accumulator (it does
        not round to nearest), u per round-to-nearest add:
          fp32 FFMA kernels            D = K + 128;
          tf32, bf16 (one wgmma pass)  D = 2 K + 128;
          3xtf32, 3xf16                D = 2 min(K, 512) + ceil(K / 128) + 128 (the wgmma
                                       accumulators are folded with RN adds every K = 128
                                       once K > 512);
        the + 128 covers the bias, the split-K partial sums and the final store.
  rep   representation error of a product: 0 for fp32; 0 for tf32 and bf16, whose reference
        is evaluated on the operands rounded as the tensor core reads them (tf32 truncated,
        bf16 round-to-nearest); 3xtf32 2^-18 (truncated hi: residuals rounded to 2^-21 each,
        dropped lo*lo <= 2^-20); 3xf16 2^-20 (11-bit hi and lo': 2^-22 per operand, dropped
        lo*lo 2^-22).
  floor 3xf16 only: an fp16 pair holds a value below 2^-14 to an absolute 2^-36 (of the scaled
        value for a gradient operand): 2^-36 (sum_k |b_k| / s_a + sum_k |a_k| / s_b).
Sums (db, dalpha) within 2^-16 of the sum of the terms' magnitudes (the BatchNorm/PReLU
convention of tests/test_bn_prelu_gpu.py) plus one fp32 rounding.  L1 loss: each fp32
difference within u |p - t|, the fp64 sum within 2^-40 of the magnitudes, the division by n
and the final fp32 rounding one ulp each.  L1 backward exact.

Memory: yfull and dx hold a huge finite guard before the kernels run and every element is
compared afterwards (an element not written fails); the slack tail of every xz buffer (read
only for GEMM rows the row map discards) holds a huge finite sentinel (2^100, or 2^15 where the
fp16 pair must stay finite) and must be unchanged; the tails of dyfull, which the 3xf16 absmax
reads, must still be exactly 0."""
import math

import pytest
import torch

import emul
from pase_b200 import gemm
from pase_b200 import functional as Fn
from pase_b200.decoder import decoder_stack
from pase_b200.losses import ContextualizedLoss
from pase_b200.minions import DecoderMinion

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 2.0 ** 100
PRECS = ["fp32", "3xtf32", "3xf16", "tf32", "bf16"]
WPLUS = dict(fmaps=[512, 256, 128], strides=[4, 4, 10], kwidths=[30, 30, 30])


# ---- comparison helpers ----
def _within(what, got, ref, tol):
    """err <= tol everywhere; -> worst err / tol."""
    err = (got.detach().double() - ref).abs()
    tol = torch.as_tensor(tol, dtype=torch.float64, device=err.device).expand_as(err)
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err - tol, torch.zeros_like(err)).reshape(-1)))
        raise AssertionError("%s: %d/%d out of bound; worst at flat %d: got %.9e ref %.9e "
                             "err %.3e tol %.3e" % (what, int(bad.sum()), bad.numel(), i,
                                                    float(got.reshape(-1)[i]),
                                                    float(ref.reshape(-1)[i]),
                                                    float(err.reshape(-1)[i]),
                                                    float(tol.reshape(-1)[i])))
    pos = tol > 0
    return float((err[pos] / tol[pos]).max()) if bool(pos.any()) else 0.0


def _ulp32(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 23)


def _report(name, ratios):
    worst = {}
    for w, r in ratios:
        worst[w] = max(worst.get(w, 0.0), r)
    print("%s: worst err / bound %s" % (name, ", ".join("%s %.3g" % kv for kv in worst.items())))


# ---- the minion ----
def make_minion(Cin, fmaps, strides, kwidths, dev, seed=0, hidden=64):
    """DecoderMinion with seeded weights (|W| ~ 1 / sqrt(fan-in)), biases and PReLU slopes in
    [-0.5, 0.5] with every fourth slope exactly 0 (the as-initialised init=0 state)."""
    m = DecoderMinion(Cin, 1, 0.0, hidden_size=hidden, hidden_layers=1, fmaps=list(fmaps),
                      strides=list(strides), kwidths=list(kwidths), loss=ContextualizedLoss("L1Loss"))
    gen = torch.Generator().manual_seed(9000 + seed)
    with torch.no_grad():
        for blk in m.blocks[:m.n_deconv]:
            W = blk.deconv.weight
            taps = -(-blk.kwidth // blk.stride)
            W.copy_(torch.randn(W.shape, generator=gen) / math.sqrt(W.shape[0] * taps))
            blk.deconv.bias.copy_(0.1 * torch.randn(W.shape[1], generator=gen))
            a = torch.rand(W.shape[1], generator=gen) - 0.5
            a[::4] = 0.0
            blk.act.weight.copy_(a)
        for p in list(m.blocks[m.n_deconv:].parameters()) + list(m.W.parameters()):
            p.copy_(torch.randn(p.shape, generator=gen) / math.sqrt(max(p[0].numel(), 1)))
    return m.to(dev)


def deconv_params(m):
    return [(blk.deconv.weight, blk.deconv.bias, blk.act.weight) for blk in m.blocks[:m.n_deconv]]


def l1_scale_grad(n_rows, C, B, L, dev, seed=0, scale=None):
    """Upstream gradient at the L1 scale: +-fp32(1 / (B L)), exact zeros at one position in 16
    (where sign(pred - target) ties); scale: an O(1) gradient instead (randn * scale)."""
    gen = torch.Generator().manual_seed(9500 + seed)
    if scale is not None:
        return (torch.randn(n_rows, C, generator=gen) * scale).to(dev)
    r = torch.randint(0, 32, (n_rows, C), generator=gen)
    c = torch.tensor(1.0 / (B * L), dtype=torch.float32)
    g = torch.where(r < 15, c, -c)
    g[r >= 30] = 0.0
    return g.to(dev)


# ---- operands as the GEMM reads them ----
def _tc(p, lda, K, ldb):
    return gemm.nt_ok(p, lda, K, ldb)


def _read(p, tc, x):
    """float64 value of an fp32 operand as the kernel multiplies it (single-pass modes round;
    the fp32-equivalent ones are compared against the fp32 value itself)."""
    if tc and p.name == "tf32":
        return emul.core._tf32_trunc(x.float()).double()
    if tc and p.name == "bf16":
        return x.float().to(torch.bfloat16).double()
    return x.double()


def _depth(p, tc, K):
    if not tc:
        return K + 128
    if p.split:
        return 2 * min(K, 512) + -(-K // 128) + 128
    return 2 * K + 128


def _rep(p, tc):
    if not tc or not p.split:
        return 0.0
    return 2.0 ** -18 if p.name == "3xtf32" else 2.0 ** -20


def _gemm_tol(p, tc, K, S, fa=None, fb=None):
    """(rep + D u) S + floor; fa + fb: sum_k |a_k| / s_b + sum_k |b_k| / s_a, broadcast over the
    output (the floor of the 3xf16 pair)."""
    tol = (_rep(p, tc) + _depth(p, tc, K) * U) * S
    if tc and p.name == "3xf16" and fa is not None:
        tol = tol + 2.0 ** -36 * (fa + fb)
    return tol


def f16_scale(dy, n):
    return emul.core.f16_grad_scale(float(dy[:n].abs().max()) * 1.0001)


# ---- float64 reference of one layer's polyphase GEMMs, from W by index arithmetic ----
def poly_weight(W, s, taps):
    """Wf[q, co, j, ci] = W[ci, co, s (taps - 1 - j) + q] (0 where the tap is >= k), float64."""
    Cin, Cout, k = W.shape
    Wp = torch.zeros(Cin, Cout, taps * s, dtype=torch.float64, device=W.device)
    Wp[:, :, :k] = W
    return Wp.view(Cin, Cout, taps, s).flip(2).permute(3, 1, 2, 0).contiguous()


def _unfold_rows(xz_s, g):
    """(b, Pd, Cin) padded input -> (b * U, taps * Cin): GEMM row u reads rows u .. u+taps-1."""
    b = xz_s.shape[0]
    v = xz_s.contiguous()
    return torch.as_strided(v, (b, g.U, g.taps * g.Cin), (g.Pd * g.Cin, g.Cin, 1)) \
        .reshape(b * g.U, g.taps * g.Cin)


def _chunks(B, rows_per_sample, budget=1 << 14):
    n = max(1, budget // max(rows_per_sample, 1))
    return [(b0, min(B, b0 + n)) for b0 in range(0, B, n)]


def fwd_gemm_checks(p, plan, i, W, b):
    """yfull[i] against the float64 polyphase product of the kernel's xz[i]."""
    g, B = plan.geoms[i], plan.B
    tc = _tc(p, g.Cin, g.taps * g.Cin, g.taps * g.Cin)
    K = g.taps * g.Cin
    Wf = poly_weight(W.detach().double(), g.s, g.taps).view(g.s * g.Cout, K)
    Wr = poly_weight(_read(p, tc, W.detach()), g.s, g.taps).view(g.s * g.Cout, K)
    bias = b.detach().double().repeat(g.s)
    xz = plan.xz[i][:B * g.Pd * g.Cin].view(B, g.Pd, g.Cin)
    y = plan.yfull[i].view(B, g.U, g.s * g.Cout)
    for b0, b1 in _chunks(B, g.U):
        X = _unfold_rows(_read(p, tc, xz[b0:b1]), g)
        ref = (X @ Wr.t() + bias).view(b1 - b0, g.U, -1)
        Xa = _unfold_rows(xz[b0:b1].double().abs(), g)
        S = (Xa @ Wf.abs().t() + bias.abs()).view(b1 - b0, g.U, -1)
        sa = Xa.sum(1).view(b1 - b0, g.U, 1)
        sb = Wf.abs().sum(1).view(1, 1, -1)
        yield ("fwd%d" % i, y[b0:b1], ref, _gemm_tol(p, tc, K, S, sb, sa))
        del X, ref, Xa, S


def crop_prelu_checks(plan, i, alpha, dst):
    """dst (B, L, C) against PReLU of the crop of yfull[i]: exact."""
    g, B = plan.geoms[i], plan.B
    C = g.Cout
    a = alpha.detach().double()
    for b0, b1 in _chunks(B, g.L):
        y = plan.yfull[i].view(B, g.U * g.s, C)[b0:b1, g.pad:g.pad + g.L].double()
        ref = torch.where(y > 0, y, (a * y).float().double())
        yield ("prelu%d" % i, dst[b0:b1], ref, 0.0)


def out_view(plan, i, out):
    """The (B, L, C) destination of layer i's crop + PReLU pass."""
    B = plan.B
    if i + 1 < len(plan.geoms):
        nx = plan.geoms[i + 1]
        return plan.xz[i + 1][:B * nx.Pd * nx.Cin].view(B, nx.Pd, nx.Cin)[:, nx.taps - 1:
                                                                           nx.taps - 1 + nx.T_in]
    g = plan.geoms[i]
    return out.view(B, g.L, g.Cout)


def pad_checks(plan):
    """The taps - 1 pad rows around every sample of xz[i] are exactly 0."""
    for i, g in enumerate(plan.geoms):
        xz = plan.xz[i][:plan.B * g.Pd * g.Cin].view(plan.B, g.Pd, g.Cin)
        pads = torch.cat([xz[:, :g.taps - 1], xz[:, g.taps - 1 + g.T_in:]], 1)
        assert bool((pads == 0).all()), "xz[%d]: pad rows not zero" % i


def bwd_checks(p, plan, i, W, b, alpha, gin, grads):
    """du, db, dalpha, the 3xf16 gradient operand, dW and dx of layer i after backward; gin:
    the (B, L, C) gradient that arrived at its output (the kernel's dx[i+1] or the upstream
    gradient); grads: (dW, db, dalpha) the parameters received."""
    g, B = plan.geoms[i], plan.B
    C, s = g.Cout, g.s
    a = alpha.detach().double()
    dyf = plan.dyfull[i]
    n_dy = B * g.U * s * C
    dy = dyf[:n_dy].view(B, g.U * s, C)
    # du and the zero margins
    assert bool((dy[:, :g.pad] == 0).all()) and bool((dy[:, g.pad + g.L:] == 0).all()), \
        "dyfull[%d]: crop margins not zero" % i
    assert bool((dyf[n_dy:] == 0).all()), "dyfull[%d]: slack tail written" % i
    S1 = torch.zeros(C, dtype=torch.float64, device=dyf.device)
    Sa1, Sal, Saa = torch.zeros_like(S1), torch.zeros_like(S1), torch.zeros_like(S1)
    for b0, b1 in _chunks(B, g.L):
        y = plan.yfull[i].view(B, g.U * s, C)[b0:b1, g.pad:g.pad + g.L].double()
        gg = gin[b0:b1].double()
        du = torch.where(y > 0, gg, (a * gg).float().double())
        yield ("du%d" % i, dy[b0:b1, g.pad:g.pad + g.L], du, 0.0)
        S1 += du.sum((0, 1))
        Sa1 += du.abs().sum((0, 1))
        t = torch.where(y > 0, torch.zeros_like(y), y * gg)
        Sal += t.sum((0, 1))
        Saa += t.abs().sum((0, 1))
        del y, gg, du, t
    dW, db, dal = grads
    yield ("db%d" % i, db, S1, 2.0 ** -16 * Sa1 + _ulp32(S1))
    yield ("dalpha%d" % i, dal, Sal, 2.0 ** -16 * Saa + _ulp32(Sal))
    K_w = g.taps * g.Cin
    tcw = gemm.tn_ok(p, s * C, g.Cin, s * C, K_w)
    tcx = gemm.nt_ok(p, s * C, g.k * C, g.k * C)
    sdy = f16_scale(dyf, dyf.numel()) if p.name == "3xf16" else 1.0
    if p.name == "3xf16" and tcw and tcx:
        op = gemm.to_operand(p, dyf, dyf.numel(), "grad")
        assert op.alpha.tolist() == [1.0 / sdy, sdy], (op.alpha.tolist(), sdy)
        for e0 in range(0, n_dy, 1 << 24):
            e1 = min(n_dy, e0 + (1 << 24))
            v = (op.hi[e0:e1].double() + op.lo[e0:e1].double() / 2048.0) / sdy
            d64 = dyf[e0:e1].double()
            yield ("dyop%d" % i, v, d64, 2.0 ** -22 * d64.abs() + 2.0 ** -36 / sdy)
            del v, d64
        del op
    # dW: sum over every sample's U GEMM rows
    xz = plan.xz[i][:B * g.Pd * g.Cin].view(B, g.Pd, g.Cin)
    dWu = torch.zeros(s * C, K_w, dtype=torch.float64, device=dyf.device)
    SW, fi, fj = torch.zeros_like(dWu), torch.zeros_like(dWu[:, :1]), torch.zeros_like(dWu[:1])
    for b0, b1 in _chunks(B, g.U * s):
        A = _read(p, tcw, dy[b0:b1]).reshape((b1 - b0) * g.U, s * C)
        X = _unfold_rows(_read(p, tcw, xz[b0:b1]), g)
        dWu += A.t() @ X
        Aa = dy[b0:b1].double().abs().reshape((b1 - b0) * g.U, s * C)
        Xa = _unfold_rows(xz[b0:b1].double().abs(), g)
        SW += Aa.t() @ Xa
        fi += Aa.sum(0)[:, None]
        fj += Xa.sum(0)[None, :] / sdy
        del A, X, Aa, Xa

    def to_w(t):        # dWu[(q, co), (j, ci)] -> dW[ci, co, s (taps - 1 - j) + q]
        t = t.view(s, C, g.taps, g.Cin).flip(2).permute(3, 1, 2, 0).reshape(g.Cin, C, g.taps * s)
        return t[:, :, :g.k]
    yield ("dW%d" % i, dW, to_w(dWu), to_w(_gemm_tol(p, tcw, B * g.U, SW, fi, fj)))
    del dWu, SW
    # dx[b, t, ci] = sum_{tap, co} dy[b, s t + tap, co] W[ci, co, tap]
    Wb = _read(p, tcx, W.detach()).permute(0, 2, 1).reshape(g.Cin, g.k * C)
    Wba = W.detach().double().abs().permute(0, 2, 1).reshape(g.Cin, g.k * C)
    dx = plan.dx[i].view(B, g.T_in, g.Cin)
    for b0, b1 in _chunks(B, g.U * s):
        d = _read(p, tcx, dy[b0:b1]).contiguous()
        A = torch.as_strided(d, (b1 - b0, g.T_in, g.k * C), (g.U * s * C, s * C, 1))
        ref = A @ Wb.t()
        da = dy[b0:b1].double().abs().contiguous()
        Aa = torch.as_strided(da, (b1 - b0, g.T_in, g.k * C), (g.U * s * C, s * C, 1))
        S = Aa @ Wba.t()
        yield ("dx%d" % i, dx[b0:b1], ref,
               _gemm_tol(p, tcx, g.k * C, S, Aa.sum(2, keepdim=True), Wba.sum(1) / sdy))
        del d, A, ref, da, Aa, S


# ---- one decoder forward + backward, every stage checked ----
def _sentinel(p):
    return 2.0 ** 15 if p.name == "3xf16" else GUARD


def decoder_case(m, B, T, dev, prec, seed=0, gscale=None):
    """Forward on one input (pads zeroed at allocation), then poison, forward on a second input
    and backward with an upstream gradient at the L1 scale (or randn * gscale); -> [(check,
    worst err / bound)]."""
    Fn.set_precision(prec)
    p = Fn.gemm_precision()
    Cin = m.num_inputs
    gen = torch.Generator().manual_seed(9100 + seed)
    x0 = torch.randn(B * T, Cin, generator=gen).to(dev)
    x = torch.randn(B * T, Cin, generator=gen).to(dev).requires_grad_(True)
    with torch.no_grad():
        decoder_stack(m, x0, B, T)
    plan = m._plans[(B, T, str(x.device))]
    pad_checks(plan)
    G = plan.geoms
    tails = []
    for i, g in enumerate(G):
        plan.yfull[i].fill_(GUARD)
        plan.dx[i].fill_(GUARD)
        t = plan.xz[i][B * g.Pd * g.Cin:]
        t.fill_(_sentinel(p))
        tails.append(t)
    params = deconv_params(m)
    for trio in params:
        for q in trio:
            q.grad = None
    out, L = decoder_stack(m, x, B, T)
    pad_checks(plan)
    for t in tails:
        assert bool((t == _sentinel(p)).all()), "xz slack tail written"
    res = []

    def run(checks):
        for (w, got, ref, tol) in checks:
            res.append((w, _within("%s %s" % (prec, w), got, ref, tol)))

    for i, (W, b, a) in enumerate(params):
        run(fwd_gemm_checks(p, plan, i, W, b))
        run(crop_prelu_checks(plan, i, a, out_view(plan, i, out)))
    C = G[-1].Cout
    dh = l1_scale_grad(B * L, C, B, L, dev, seed, gscale)
    out.backward(dh)
    for i in range(len(G) - 1, -1, -1):
        W, b, a = params[i]
        g = G[i]
        gin = dh.view(B, L, C) if i + 1 == len(G) else plan.dx[i + 1].view(B, g.L, g.Cout)
        run(bwd_checks(p, plan, i, W, b, a, gin, (W.grad, b.grad, a.grad)))
    assert torch.equal(x.grad, plan.dx[0].view(B * T, Cin))
    return res


@pytest.fixture()
def precision(monkeypatch):
    monkeypatch.setattr(Fn, "PRECISION", Fn.PRECISION)       # restored after the test
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    print("peak device memory %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9))
    torch.cuda.empty_cache()


def test_workers_plus_geometry():
    """The shapes named in the module docstring."""
    m = make_minion(256, WPLUS["fmaps"], WPLUS["strides"], WPLUS["kwidths"], "cpu")
    from pase_b200.decoder import DecoderPlan
    layers = [(blk.deconv.weight.shape[0], blk.deconv.weight.shape[1], blk.kwidth, blk.stride,
               blk.pad) for blk in m.blocks[:m.n_deconv]]
    plan = DecoderPlan(layers, 32, 200, torch.device("meta"))
    got = [(g.Cin, g.Cout, g.k, g.s, g.pad, g.taps, g.T_in, g.L, g.U) for g in plan.geoms]
    assert got == [(256, 512, 30, 4, 13, 8, 200, 800, 207),
                   (512, 256, 30, 4, 13, 8, 800, 3200, 807),
                   (256, 128, 30, 10, 10, 3, 3200, 32000, 3202)], got


@pytest.mark.parametrize("prec", PRECS)
def test_workers_plus_stages(prec, precision):
    """B = 32, T' = 200, the workers+ decoder, upstream gradient at the L1 scale."""
    m = make_minion(256, WPLUS["fmaps"], WPLUS["strides"], WPLUS["kwidths"], "cuda", seed=1)
    _report("decoder workers+ B=32 T'=200 %s" % prec, decoder_case(m, 32, 200, "cuda", prec))


def test_workers_plus_stages_unit_gradient(precision):
    """An O(1) upstream gradient (no fp16 scaling regime) in the default precision."""
    m = make_minion(256, WPLUS["fmaps"], WPLUS["strides"], WPLUS["kwidths"], "cuda", seed=2)
    _report("decoder workers+ O(1) gradient 3xf16",
            decoder_case(m, 32, 200, "cuda", "3xf16", seed=2, gscale=1.0))


# geometry edges at tensor-core widths: (Cin, fmaps, strides, kwidths, B, T)
EDGES = {
    "k<s": (64, [128], [4], [2], 3, 9),
    "k==s-default": (256, [256, 256, 128, 128, 128, 64], [2, 2, 2, 2, 2, 5],
                     [2, 2, 2, 2, 2, 5], 2, 5),
    "k%s==0": (128, [64, 128], [4, 3], [8, 9], 3, 11),
    "T_in=1": (256, [128, 64], [4, 10], [30, 30], 4, 1),
    "B=1": (256, [128, 128], [4, 10], [30, 30], 1, 13),
    "ffma-96": (96, [96, 64], [4, 10], [30, 30], 2, 6),
}


@pytest.mark.parametrize("prec", ["fp32", "3xtf32", "3xf16"])
@pytest.mark.parametrize("edge", list(EDGES))
def test_geometry_edges(edge, prec, precision):
    Cin, fm, st, kw, B, T = EDGES[edge]
    m = make_minion(Cin, fm, st, kw, "cuda", seed=len(edge))
    p = gemm.PRECISIONS[prec]
    if edge == "ffma-96":            # 96 channels: the 16-bit formats fall back to FFMA
        assert not gemm.nt_ok(p, 96, 8 * 96, 8 * 96) or p.fmt != gemm.FMT_F16X2
        assert not gemm.tn_ok(p, 4 * 96, 96, 4 * 96, 8 * 96) or p.fmt != gemm.FMT_F16X2
        assert gemm.nt_ok(gemm.PRECISIONS["3xtf32"], 96, 8 * 96, 8 * 96)
    _report("decoder %s %s" % (edge, prec), decoder_case(m, B, T, "cuda", prec, seed=3))


# ---- the rest of the worker at full rate: MLP, output layer, L1 ----
def test_worker_tail_full_rate(precision):
    """B = 32, L = 32000: linear_rows 128 -> 64, prelu_rows, the 64 -> 1 output layer (ldo one
    128-byte row, padding columns zero), ContextualizedLoss('L1Loss') and its backward, the
    output layer's dW / db over 1,024,000 rows."""
    Fn.set_precision("3xf16")
    p = Fn.gemm_precision()
    from pase_b200.minions import rows_to_pred
    B, L, dev = 32, 32000, "cuda"
    n = B * L
    m = make_minion(256, WPLUS["fmaps"], WPLUS["strides"], WPLUS["kwidths"], dev, seed=4)
    blk = m.blocks[m.n_deconv]
    gen = torch.Generator().manual_seed(9700)
    h = torch.randn(n, 128, generator=gen).abs().to(dev)          # post-PReLU-like rows
    res = []
    u = Fn.linear_rows(h, blk.W.weight, blk.W.bias)
    W1, b1 = blk.W.weight.detach().double().view(64, 128), blk.W.bias.detach().double()
    tc = gemm.nt_ok(p, 128, 128, 128)
    h64 = h.double()
    res.append(("hidden", _within("hidden", u[:, :64], h64 @ W1.t() + b1,
                                  _gemm_tol(p, tc, 128, h64 @ W1.abs().t() + b1.abs(),
                                            W1.abs().sum(1), h64.sum(1, keepdim=True)))))
    del h64, h
    hh = Fn.prelu_rows(u, blk.act.weight, 64)[:, :64]
    a1 = blk.act.weight.detach().double()
    u64 = u[:, :64].double()
    res.append(("prelu", _within("prelu", hh, torch.where(u64 > 0, u64, (a1 * u64).float()
                                                          .double()), 0.0)))
    hh = hh.detach().requires_grad_(True)
    y = Fn.linear_rows(hh, m.W.weight, m.W.bias)
    ldo = y.shape[1]
    assert ldo == p.eb and bool((y[:, 1:] == 0).all()), "output padding columns not zero"
    W2, b2 = m.W.weight.detach().double().view(1, 64), m.W.bias.detach().double()
    tc2 = gemm.nt_ok(p, 64, 64, 64)
    h64 = hh.detach().double()
    res.append(("out", _within("out", y[:, :1], h64 @ W2.t() + b2,
                               _gemm_tol(p, tc2, 64, h64.abs() @ W2.abs().t() + b2.abs(),
                                         W2.abs().sum(1), h64.abs().sum(1, keepdim=True)))))
    # target: pred + noise, exact ties at one position in 16
    pred = y[:, 0].detach()
    tgt = pred + 0.3 * torch.randn(n, generator=gen).to(dev)
    tgt[::16] = pred[::16]
    grab = {}
    y.register_hook(lambda g: grab.setdefault("dy", g))
    loss = ContextualizedLoss("L1Loss")(rows_to_pred(y, B, L, 1), tgt.view(B, 1, L))
    d = (pred.double() - tgt.double()).abs()
    ref = d.sum() / n
    tol = (U * d.sum() + 2.0 ** -40 * d.sum()) / n + 2 * _ulp32(ref)
    res.append(("l1", _within("l1", loss.reshape(()), ref, tol)))
    loss.backward()
    dy = grab["dy"]
    k = torch.tensor(1.0 / n, dtype=torch.float32).item()
    diff = pred - tgt
    want = torch.where(diff > 0, k, torch.where(diff < 0, -k, 0.0))
    assert bool((want[::16] == 0).all())
    assert torch.equal(dy[:, 0], want), "L1 backward not exactly +-fp32(1/n) / 0 at ties"
    assert bool((dy[:, 1:] == 0).all())
    # output layer weight and bias gradients over every row
    d64 = dy[:, 0].double()
    tcw = gemm.tn_ok(p, ldo, 64, ldo, 64)
    sdy = f16_scale(dy.reshape(-1), dy.numel()) if tcw else 1.0
    S = d64.abs() @ h64.abs()
    res.append(("dW_out", _within("dW_out", m.W.weight.grad.view(64), d64 @ h64,
                                  _gemm_tol(p, tcw, n, S, d64.abs().sum(), h64.abs().sum(0) / sdy))))
    res.append(("db_out", _within("db_out", m.W.bias.grad, d64.sum(),
                                  2.0 ** -16 * d64.abs().sum() + _ulp32(d64.sum()))))
    _report("worker tail B=32 L=32000 3xf16", res)


# ---- host behaviour ----
def test_second_forward_before_backward_raises(precision):
    Fn.set_precision("3xf16")
    m = make_minion(64, [64, 64], [4, 10], [30, 30], "cuda", seed=5)
    x = torch.randn(2 * 5, 64, device="cuda", requires_grad=True)
    out, L = decoder_stack(m, x, 2, 5)
    decoder_stack(m, x.detach() * 2, 2, 5)
    with pytest.raises(RuntimeError, match="overwritten"):
        out.backward(torch.ones_like(out))


def test_plan_cache_three_keys(precision):
    """The cache keeps two plans: (B, T) keys used in turn each still give the results of a
    fresh minion (bit-equal: the kernels are deterministic)."""
    Fn.set_precision("3xf16")
    m = make_minion(64, [64, 64], [4, 10], [30, 30], "cuda", seed=6)
    keys = [(2, 5), (3, 4), (1, 7), (2, 5), (1, 7), (3, 4)]
    gen = torch.Generator().manual_seed(9800)
    xs = {k: torch.randn(k[0] * k[1], 64, generator=gen).cuda() for k in set(keys)}
    for k in keys:
        outs = []
        for mm in (m, make_minion(64, [64, 64], [4, 10], [30, 30], "cuda", seed=6)):
            x = xs[k].clone().requires_grad_(True)
            out, L = decoder_stack(mm, x, *k)
            out.backward(torch.ones_like(out))
            outs.append((out.detach().clone(), x.grad.clone(),
                         [q.grad.clone() for trio in deconv_params(mm) for q in trio]))
            for q in mm.parameters():
                q.grad = None
        assert len(m._plans) <= 2
        (o0, g0, w0), (o1, g1, w1) = outs
        assert torch.equal(o0, o1) and torch.equal(g0, g1), k
        assert all(torch.equal(a, b) for a, b in zip(w0, w1)), k
