"""The waveform gradient of WaveFe on the GPU (DESIGN.md section 17): the sinc-layer input
gradient kernels alone against float64 computed from their own inputs, dx end to end against
the float64 oracle, the invariants of the data-gradient-only sweep in every precision, and dx
through WaveFe.forward."""
import pytest
import torch
import torch.nn.functional as F

import pase_oracle as O
from helpers import resolve_cfg, fill_state_dict, seeded_randn, rel_l2
from pase_b200 import encoder as enc
from pase_b200.frontend import WaveFe

pytestmark = pytest.mark.gpu

PASEP = "cfg/frontend/PASE+.cfg"
PASE = "cfg/frontend/PASE.cfg"
PRECISIONS = ["fp32", "3xtf32", "tf32", "bf16", "3xf16"]


def _native(cfg_name, seed, training, precision, frozen=False):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.load_state_dict(fill_state_dict(m.state_dict(), seed))
    m.precision = precision
    m = m.cuda().train(training)
    if frozen:
        m.requires_grad_(False)
    return m


def _dx(model, x, cot):
    xr = x.detach().clone().requires_grad_(True)
    y = model(xr)
    (y * cot).sum().backward()
    torch.cuda.synchronize()
    return y.detach(), xr.grad


# -- the kernels alone ---------------------------------------------------------------------
# per output, |error| <= c * sum |dy| |filt| over its products: the fp32-equivalent modes sum
# 16064 (fold 4) .. 20480 (fold 64) products in fp32 (FFMA, or fp32 flushes of the tensor-core
# accumulators every 128 k); tf32 truncates both operands to 10 mantissa bits; bf16 stores dy in
# bf16 (exact here: the reference reads the stored value) and rounds the bank to 8 bits.
KERNEL_BOUND = {"fp32": 2.0 ** -14, "3xtf32": 2.0 ** -14, "3xf16": 2.0 ** -14,
                "tf32": 2.0 ** -9, "bf16": 2.0 ** -7}


def _dy_float64(plan, g):
    """The sinc layer's output gradient as the GEMM reads it: plan.dyz[0] (per sample Ty frames
    x C channels), descaled, as (N, C, T_out) float64."""
    N, C, p = plan.N, g.Cout, plan.precision
    n = N * g.Ty * C
    hi = plan.dyz[0][:n]
    if p.name == "3xf16":
        v = hi.double() + plan.dyz_lo[0][:n].double() / 2048.0
        v = v * float(plan.gscale[0][0])
    else:
        v = hi.double()
    return v.view(N, g.Ty, C)[:, :g.T_out].permute(0, 2, 1)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("N,T", [(32, 32000), (1, None), (3, 32000 + 37)])
def test_sinc_input_grad_kernels(precision, N, T):
    """pase_sinc_make (bank), pase_sinc_dgrad_weight, pase_sinc_dgrad_pack, the polyphase GEMM
    and pase_reflect_fold_wave together, on the dy a frozen PASE+ backward left in dyz[0]:
    against conv_transpose1d + the reflect adjoint in float64 of that dy and bank.  The output
    and dxpad[0] are filled with NaN first (an element left unwritten fails); dyz[0] is read
    only.  T None: the encoder's minimum length."""
    model = _native(PASEP, 41, True, precision, frozen=True)
    if T is None:
        T = enc.min_length(model.cfg)
    x = seeded_randn((N, 1, T), 42, 0.5).cuda()
    y, dx0 = _dx(model, x, seeded_randn((N, 256, model.frame_counts(T)[-1]), 43).cuda())
    plan = model._plan(N, T, x.device)
    g = plan.geoms[0]
    dyz = plan.dyz[0].clone()
    dyz_lo = None if plan.dyz_lo[0] is None else plan.dyz_lo[0].clone()
    dx = torch.full((N, 1, T), float("nan"), device="cuda")
    plan.dxpad[0].fill_(float("nan"))
    params = dict(model.named_parameters())
    enc._sinc_input_grad(plan, model, lambda k: params[k].detach().reshape(-1), g, dx)
    torch.cuda.synchronize()
    assert torch.equal(plan.dyz[0], dyz) and (dyz_lo is None or torch.equal(plan.dyz_lo[0], dyz_lo))
    assert torch.isfinite(dx).all()
    assert torch.equal(dx, dx0)                  # the same launches as inside the backward
    dy = _dy_float64(plan, g)
    filt = plan.filt.double().view(g.Cout, 1, g.k)
    fold = lambda d: (d[:, 0, g.padL:g.padL + T].clone()
                      .index_add_(1, torch.arange(1, g.padL + 1, device="cuda"),
                                  d[:, 0, :g.padL].flip(1))
                      .index_add_(1, torch.arange(T - 1 - g.padR, T - 1, device="cuda"),
                                  d[:, 0, g.padL + T:].flip(1)))
    ref = fold(F.conv_transpose1d(dy, filt))
    mag = fold(F.conv_transpose1d(dy.abs(), filt.abs()))
    err = (dx[:, 0].double() - ref).abs()
    bound = KERNEL_BOUND[precision] * mag + 1e-30
    worst = float((err / bound).max())
    print("%s N=%d T=%d: worst |err| / bound = %.3f, rel-L2 %.2e"
          % (precision, N, T, worst, rel_l2(dx[:, 0], ref)))
    assert worst <= 1.0


# -- end to end against the float64 oracle --------------------------------------------------
_REF = {}


def _oracle(cfg_name, seed, N, T, training, dtype):
    """dL/dx of L = sum(y * cot) through the oracle (plain torch, on the device; TF32 off)."""
    key = (cfg_name, seed, N, T, training, dtype)
    if key not in _REF:
        cfg = resolve_cfg(cfg_name)
        sd = fill_state_dict(WaveFe(**cfg).state_dict(), seed)
        sd = {k: (v.to("cuda", dtype) if v.is_floating_point() else v.cuda()) for k, v in sd.items()}
        x = seeded_randn((N, 1, T), seed + 1, 0.5).cuda()
        xx = x.to(dtype).requires_grad_(True)
        allow = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            y = O.encoder_forward(xx, sd, cfg, training=training)
            cot = seeded_randn(tuple(y.shape), seed + 2).cuda()
            (y * cot.to(dtype)).sum().backward()
        finally:
            torch.backends.cudnn.allow_tf32 = allow
        _REF[key] = (x, cot, xx.grad.double())
    return _REF[key]


# floor of the relative L2 bound: a flipped PReLU gate moves dx coherently below it, as it moves
# the parameter gradients (test_encoder_gpu.test_benchmark_shape_against_oracle uses 2e-3 for
# them); the float32 oracle's own error is measured in the same run and printed
FLOOR = 2e-3


@pytest.mark.parametrize("cfg_name,training,frozen,precision", [
    (PASEP, True, False, "3xf16"), (PASEP, True, False, "3xtf32"),
    (PASEP, False, True, "3xf16"), (PASE, False, True, "3xf16"),
    (PASEP, True, False, "tf32"), (PASEP, True, False, "bf16")])
def test_dx_against_oracle(cfg_name, training, frozen, precision):
    """B=32, T=32000.  fp32-equivalent modes: rel-L2 to the float64 oracle within max(2 x the
    float32 oracle's own error, FLOOR); tf32 within 10 x that; bf16: cosine > 0.98."""
    seed, N, T = 51, 32, 32000
    x, cot, d64 = _oracle(cfg_name, seed, N, T, training, torch.float64)
    _, _, d32 = _oracle(cfg_name, seed, N, T, training, torch.float32)
    model = _native(cfg_name, seed, training, precision, frozen)
    _, dx = _dx(model, x, cot)
    e_nat, e_ref = rel_l2(dx.double(), d64), rel_l2(d32, d64)
    cos = float(F.cosine_similarity(dx.double().reshape(1, -1), d64.reshape(1, -1)))
    print("%s %s train=%s frozen=%s: dx rel-L2 native %.2e, fp32 oracle %.2e, cosine %.6f"
          % (cfg_name, precision, training, frozen, e_nat, e_ref, cos))
    if precision == "bf16":
        assert cos > 0.98
    elif precision == "tf32":
        assert e_nat <= 10 * max(2 * e_ref, FLOOR)
    else:
        assert e_nat <= max(2 * e_ref, FLOOR)


# -- invariants ----------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
def test_input_grad_invariants(precision):
    """Outputs and every parameter gradient bit-equal with and without x.requires_grad; a frozen
    encoder's dx bit-equal to the full sweep's and run to run; no .grad on a frozen encoder."""
    N, T = 4, 16000
    x = seeded_randn((N, 1, T), 61, 0.5).cuda()
    model = _native(PASEP, 60, True, precision)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    cot = seeded_randn((N, 256, T // 160), 62).cuda()

    def run(x_grad, frozen):
        model.load_state_dict(state)
        model.zero_grad(set_to_none=True)
        model.requires_grad_(not frozen)
        xr = x.clone().requires_grad_(x_grad)
        y = model(xr)
        (y * cot).sum().backward()
        torch.cuda.synchronize()
        return y.detach(), {k: p.grad for k, p in model.named_parameters()}, xr.grad

    y0, g0, _ = run(False, False)
    y1, g1, dx_full = run(True, False)
    assert torch.equal(y0, y1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    _, gf, dx_a = run(True, True)
    assert all(v is None for v in gf.values())
    _, _, dx_b = run(True, True)
    assert torch.equal(dx_a, dx_full) and torch.equal(dx_a, dx_b)
    assert torch.isfinite(dx_a).all() and float(dx_a.abs().max()) > 0


# -- the public surface --------------------------------------------------------------------
def test_dx_through_forward_batches():
    """WaveFe.forward with a dict batch and with the chunk_rand triplet: every input tensor gets
    its part of the dx of the concatenated batch."""
    model = _native(PASEP, 71, True, "3xf16")
    N, T = 2, 16000
    parts = {k: seeded_randn((N, 1, T), 72 + i, 0.5).cuda()
             for i, k in enumerate(("chunk", "chunk_ctxt", "chunk_rand"))}
    cat = torch.cat(list(parts.values()), 0)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    cot = seeded_randn((3 * N, 256, T // 160), 75).cuda()
    _, ref = _dx(model, cat, cot)
    model.load_state_dict(state)
    leaves = {k: v.clone().requires_grad_(True) for k, v in parts.items()}
    emb, _ = model(dict(leaves))                 # the triplet: (per-key embeddings, chunk's)
    (torch.cat(emb, 0) * cot).sum().backward()
    for i, k in enumerate(leaves):
        assert torch.equal(leaves[k].grad, ref[i * N:(i + 1) * N]), k
    model.load_state_dict(state)
    _, ref1 = _dx(model, parts["chunk"], cot[:N])
    model.load_state_dict(state)
    leaf = parts["chunk"].clone().requires_grad_(True)
    y, _ = model({"chunk": leaf})
    (y * cot[:N]).sum().backward()
    assert torch.equal(leaf.grad, ref1)


def test_frozen_encoder_as_feature_loss():
    """The perceptual-loss set-up: a frozen eval-mode PASE+ as an L1 feature loss on the output
    of a trainable nn.Conv1d; the target forward runs first, under no_grad.  The upstream
    layer's weight gradient against the same computation in float64 through the oracle."""
    seed, N, T = 81, 2, 16000
    model = _native(PASEP, seed, False, "3xf16", frozen=True)
    up = torch.nn.Conv1d(1, 1, 9, padding=4).cuda()
    with torch.no_grad():
        up.weight.copy_(seeded_randn((1, 1, 9), seed + 1, 0.3))
        up.weight[0, 0, 4] += 1.0
        up.bias.zero_()
    clean = seeded_randn((N, 1, T), seed + 2, 0.5).cuda()
    noisy = clean + seeded_randn((N, 1, T), seed + 3, 0.05).cuda()
    with torch.no_grad():
        ref = model(clean)
    loss = (model(up(noisy)) - ref).abs().mean()
    loss.backward()
    assert all(p.grad is None for p in model.parameters())

    cfg = resolve_cfg(PASEP)
    sd = {k: (v.double() if v.is_floating_point() else v)
          for k, v in model.state_dict().items()}
    w64 = up.weight.detach().double().requires_grad_(True)
    b64 = up.bias.detach().double().requires_grad_(True)
    ref64 = O.encoder_forward(clean.double(), sd, cfg, training=False)
    y64 = O.encoder_forward(F.conv1d(noisy.double(), w64, b64, padding=4), sd, cfg,
                            training=False)
    (y64 - ref64).abs().mean().backward()
    e_w, e_b = rel_l2(up.weight.grad, w64.grad), rel_l2(up.bias.grad, b64.grad)
    print("upstream conv gradient rel-L2: weight %.2e, bias %.2e" % (e_w, e_b))
    # L1: sign(y - ref) flips where the two runs' features straddle the target
    assert e_w < 1e-2 and e_b < 1e-2
