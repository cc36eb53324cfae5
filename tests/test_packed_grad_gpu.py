"""WaveFe.encode_packed on one H100 (DESIGN.md section 18): the forward is extract's, each
utterance's waveform gradient is that of its own B=1 encode, the parameter gradients are the
sum of the B=1 ones, the frozen sweep, grad_sink, allocations after warm-up and extract left
as it was."""
import pytest
import torch

import pase_oracle as O
from helpers import resolve_cfg, fill_state_dict, seeded_randn, rel_l2
from pase_b200.frontend import WaveFe

pytestmark = pytest.mark.gpu

LENGTHS = [471, 1000, 1763, 3200, 4001, 12345, 16000, 16001, 31999, 48000, 82081, 100000]
PRECISIONS = ["fp32", "tf32", "3xtf32", "3xf16", "bf16"]
CONFIGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
# relative L2 between the packed parameter gradients and the sum of the B=1 ones (summation
# order over the utterances differs; bf16 / tf32 also round the operands)
PARAM_TOL = {"fp32": 1e-4, "3xtf32": 1e-4, "3xf16": 1e-3, "tf32": 1e-2, "bf16": 5e-2}


def _model(cfg_name, precision):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.precision = precision
    m.load_state_dict(fill_state_dict(m.state_dict(), 11))
    return m.cuda().eval()


def _corpus(lengths, seed=5):
    return [seeded_randn((T,), seed + i, 0.5).cuda() for i, T in enumerate(lengths)]


def _packed(m, wavs, cots):
    xs = [w.clone().requires_grad_(True) for w in wavs]
    m.zero_grad(set_to_none=True)
    ys = m.encode_packed(xs)
    sum((y * c).sum() for y, c in zip(ys, cots)).backward()
    return ys, [x.grad for x in xs], {k: p.grad.clone() for k, p in m.named_parameters()
                                      if p.grad is not None}


def _single(m, w, cot):
    x = w.view(1, 1, -1).clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    y, _ = m.encode(x)
    (y * cot).sum().backward()
    return x.grad.view(-1), {k: p.grad.clone() for k, p in m.named_parameters()
                             if p.grad is not None}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", CONFIGS)
def test_packed_grad_matches_single(name, precision):
    m = _model(name, precision)
    wavs = _corpus(LENGTHS)
    with torch.no_grad():
        ref = m.extract(wavs)
    cots = [seeded_randn(tuple(y.shape), 40 + i).cuda() for i, y in enumerate(ref)]
    ys, dxs, grads = _packed(m, wavs, cots)
    for y, r in zip(ys, ref):
        assert torch.equal(y.detach(), r)
    psum, worst = {}, 0.0
    for i, (w, c) in enumerate(zip(wavs, cots)):
        dx1, g1 = _single(m, w, c)
        if precision == "3xf16":
            worst = max(worst, rel_l2(dxs[i], dx1))
        else:
            assert torch.equal(dxs[i], dx1), (i, rel_l2(dxs[i], dx1))
        for k, v in g1.items():
            psum[k] = v if k not in psum else psum[k] + v
    if precision == "3xf16":
        print("3xf16 dx rel-L2 max %.3e" % worst)
        assert worst < 1e-4
    pw = max(rel_l2(grads[k], v) for k, v in psum.items() if float(v.norm()) > 0)
    print("%s %s param grad rel-L2 max %.3e" % (name, precision, pw))
    assert pw < PARAM_TOL[precision]


@pytest.mark.parametrize("precision", ["3xf16", "bf16"])
def test_frozen_sweep_and_sink(precision):
    m = _model(CONFIGS[1], precision)
    wavs = _corpus([471, 16001, 82081, 3200])
    with torch.no_grad():
        ref = m.extract(wavs)
    cots = [seeded_randn(tuple(y.shape), 60 + i).cuda() for i, y in enumerate(ref)]
    _, dx_full, grads = _packed(m, wavs, cots)
    for _, p in m.named_parameters():
        p.requires_grad_(False)
    runs = [_packed(m, wavs, cots)[1] for _ in range(2)]
    for a, b, c in zip(dx_full, *runs):
        assert torch.equal(a, b) and torch.equal(b, c)
    for _, p in m.named_parameters():
        p.requires_grad_(True)
    from pase_b200.optim import FlatAdam
    opt = FlatAdam([p for _, p in m.named_parameters()], lr=1e-3).bind_encoder(m)
    opt.zero_grad(set_to_none=True)
    xs = [w.clone().requires_grad_(True) for w in wavs]
    sum((y * c).sum() for y, c in zip(m.encode_packed(xs), cots)).backward()
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, grads[k]), k
    m.grad_sink = None


def test_extract_unchanged():
    m = _model(CONFIGS[1], "3xf16")
    wavs = _corpus([471, 16001, 3200])
    with torch.no_grad():
        ref = [y.clone() for y in m.extract(wavs)]
    nb = [p.nbytes() for p in m._packed_plans.values()]
    _packed(m, wavs, [torch.ones_like(y) for y in ref])
    with torch.no_grad():
        again = m.extract(wavs)
    for a, b in zip(again, ref):
        assert torch.equal(a, b)
    assert [p.nbytes() for p in m._packed_plans.values()] == nb


def test_feature_loss_end_to_end():
    """A frozen PASE+ as an L1 feature loss on a trainable Conv1d over mixed lengths."""
    m = _model(CONFIGS[1], "3xf16").requires_grad_(False)
    net = torch.nn.Conv1d(1, 1, 9, padding=4).cuda()
    wavs = _corpus([471, 16001, 48000, 3200])
    targets = [w * 0.5 for w in wavs]
    with torch.no_grad():
        tfeat = m.extract(targets)
    net.zero_grad()
    outs = [net(w.view(1, 1, -1)).view(-1) for w in wavs]
    loss = sum((y - t).abs().mean() for y, t in zip(m.encode_packed(outs), tfeat))
    loss.backward()
    g_packed = net.weight.grad.clone()
    net.zero_grad()
    for w, t in zip(wavs, tfeat):
        y, _ = m.encode(net(w.view(1, 1, -1)))
        (y - t).abs().mean().backward()
    assert rel_l2(g_packed, net.weight.grad) < 1e-3


def _r512(nbytes):
    return -(-nbytes // 512) * 512          # the caching allocator's block granularity


@pytest.mark.parametrize("frozen", [False, True])
def test_allocations_after_warmup(frozen):
    """After warm-up a call keeps nothing allocated but its outputs (one buffer), the packed dx
    and, in the full sweep, the parameter gradients: at most one block per parameter, the cast
    vector of the small gradients and the conv weight-gradient buffer."""
    m = _model(CONFIGS[1], "3xf16")
    for _, p in m.named_parameters():
        p.requires_grad_(not frozen)
    wavs = _corpus([471, 16001, 82081, 3200])
    with torch.no_grad():
        cots = [torch.randn_like(y) for y in m.extract(wavs)]
    for _ in range(2):
        _packed(m, wavs, cots)
    m.zero_grad(set_to_none=True)
    xs = [w.clone().requires_grad_(True) for w in wavs]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    ys = m.encode_packed(xs)
    sum((y * c).sum() for y, c in zip(ys, cots)).backward()
    torch.cuda.synchronize()
    bound = _r512(sum(y.numel() for y in ys) * 4) + _r512(sum(w.numel() for w in wavs) * 4)
    if not frozen:
        plan = next(iter(m._grad_plans.values()))
        params = [p for _, p in m.named_parameters()]
        bound += sum(_r512(p.numel() * 4) for p in params) + _r512(plan.grad_vec.numel() * 4)
        bound += _r512(sum(p.numel() * 4 for n, p in m.named_parameters()
                           if n.endswith("conv.weight") and p.dim() == 3))
        assert all(p.grad is not None for p in params)
    grew = torch.cuda.memory_allocated() - base
    print("frozen=%s: %d bytes kept, bound %d" % (frozen, grew, bound))
    assert grew <= bound


@pytest.mark.parametrize("precision", ["fp32", "3xf16", "bf16"])
def test_zero_rows_rewritten_on_device(precision):
    """The rows of the backward layout outside the valid frames are rewritten as zero on every
    call: after a call with one order, the gradient buffers filled with NaN and a call with the
    offsets moved gives the bits of a fresh model's call."""
    wavs = _corpus([471, 16001, 82081, 3200, 1000])
    order = [3, 0, 4, 2, 1]
    used, fresh = _model(CONFIGS[1], precision), _model(CONFIGS[1], precision)
    with torch.no_grad():
        ref = fresh.extract([wavs[i] for i in order])
    cots = [seeded_randn(tuple(y.shape), 80 + i).cuda() for i, y in enumerate(ref)]
    with torch.no_grad():
        first = used.extract(wavs)
    _packed(used, wavs, [torch.ones_like(y) for y in first])
    plan = next(iter(used._grad_plans.values()))
    for t in plan.dyz + plan.dyz_lo + [plan.dYg]:
        if t is not None:
            t.fill_(float("nan"))
    _, dx_used, g_used = _packed(used, [wavs[i] for i in order], cots)
    _, dx_fresh, g_fresh = _packed(fresh, [wavs[i] for i in order], cots)
    for a, b in zip(dx_used, dx_fresh):
        assert torch.equal(a, b)
    for k, v in g_fresh.items():
        assert torch.isfinite(g_used[k]).all() and rel_l2(g_used[k], v) < 1e-6, k


def _oracle_pack(m, wavs, cots, dtype):
    """Per-utterance dx (concatenated) and summed parameter gradients of sum_i <y_i, cot_i>
    through the oracle in `dtype` (plain torch on the device, TF32 off)."""
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    leaves = {k: sd[k].clone().requires_grad_(True) for k, _ in m.named_parameters()}
    sd.update(leaves)
    allow = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    dxs = []
    try:
        for w, c in zip(wavs, cots):
            x = w.to(dtype).view(1, 1, -1).requires_grad_(True)
            (O.encoder_forward(x, sd, m.cfg, training=False) * c.to(dtype)).sum().backward()
            dxs.append(x.grad.view(-1))
    finally:
        torch.backends.cudnn.allow_tf32 = allow
    return torch.cat(dxs), {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("precision", ["3xf16", "3xtf32"])
def test_benchmark_scale_against_float64_oracle(precision):
    """32 utterances around 32000 samples (1.024 M in one pack) against the float64 oracle, with
    the bound of the uniform backward at B=32, T=32000 (tests/test_input_grad_gpu.py): the
    pack's dx within max(2 x the float32 oracle's own error, 2e-3) relative L2, the summed
    parameter gradients within 2e-3 (tests/test_encoder_gpu.py)."""
    g = torch.Generator().manual_seed(9)
    d = (torch.randint(-8000, 8001, (16,), generator=g)).tolist()
    lens = [32000 + x for x in d] + [32000 - x for x in d]
    m = _model(CONFIGS[1], precision)
    wavs = _corpus(lens, seed=70)
    with torch.no_grad():
        ref = m.extract(wavs)
    cots = [seeded_randn(tuple(y.shape), 90 + i).cuda() for i, y in enumerate(ref)]
    _, dxs, grads = _packed(m, wavs, cots)
    d64, p64 = _oracle_pack(m, wavs, cots, torch.float64)
    d32, _ = _oracle_pack(m, wavs, cots, torch.float32)
    e_dx, e_ref = rel_l2(torch.cat(dxs), d64), rel_l2(d32, d64)
    worst_p = max(rel_l2(grads[k], v) for k, v in p64.items() if float(v.norm()) > 0)
    print("%s B=32 scale: dx rel-L2 %.2e (float32 oracle %.2e), parameter gradients %.2e"
          % (precision, e_dx, e_ref, worst_p))
    assert e_dx <= max(2 * e_ref, 2e-3)
    assert worst_p < 2e-3
