"""WaveFe.encode_long on one H100 (DESIGN.md section 20): features equal to extract_long, the
waveform and parameter gradients against the whole-recording backward of encode and against the
float64 oracle, a 40 M-sample recording that encode refuses (bounded memory, two windows, two
runs), and grad_sink through FlatAdam."""
import pytest
import torch

import pase_oracle as O
from helpers import resolve_cfg, fill_state_dict, seeded_randn, rel_l2
from pase_b200 import encoder as enc
from pase_b200.frontend import WaveFe

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "3xtf32", "3xf16", "bf16"]
CONFIGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
# relative L2 of dx and of each parameter gradient against the whole-recording backward: the
# summation order differs at the seams and in the weight-gradient reductions; tf32 / bf16 also
# round operands whose values differ in the last bit (measured on an H100: at most 1.3e-6 in
# fp32, 3xtf32 and 3xf16, 2.1e-4 in tf32, 1.2e-3 in bf16; DESIGN.md section 20)
TOL = {"fp32": 1e-5, "3xtf32": 1e-5, "3xf16": 1e-5, "tf32": 1e-3, "bf16": 5e-3}


def _model(cfg_name, precision):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.precision = precision
    m.load_state_dict(fill_state_dict(m.state_dict(), 11))
    return m.cuda().eval()


def _grads(m):
    return {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}


def _clear(m):
    for _, p in m.named_parameters():
        p.grad = None


def _long(m, x, cot, window):
    xl = x.clone().requires_grad_(True)
    _clear(m)
    y = m.encode_long(xl, window)
    (y * cot).sum().backward()
    return y, xl.grad, _grads(m)


@pytest.mark.parametrize("window", ["min", 1 << 19])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg_name", CONFIGS)
def test_against_whole_recording(cfg_name, precision, window):
    m = _model(cfg_name, precision)
    win = enc.min_window(m.cfg) if window == "min" else window
    L = 1_200_000 + 37
    x = seeded_randn((L,), 17, 0.5).cuda()
    with torch.no_grad():
        feats = m.extract_long(x, window=win)
    cot = seeded_randn(tuple(feats.shape), 18).cuda()
    y, dx, grads = _long(m, x, cot, win)
    assert torch.equal(y, feats)
    xw = x.clone().view(1, 1, -1).requires_grad_(True)
    _clear(m)
    yw, _ = m.encode(xw)
    (yw * cot).sum().backward()
    dxw, gw = xw.grad.view(-1), _grads(m)
    err = {k: rel_l2(grads[k], v) for k, v in gw.items() if float(v.norm()) > 0}
    # samples whose gradient comes from one crop only: away from every seam's overlap
    hop, segs = enc.hop_size(m.cfg), enc.plan_windows(m.cfg, L, win)
    single = torch.ones(L, dtype=torch.bool, device=x.device)
    for a, b in zip(segs[:-1], segs[1:]):
        single[b["seg_start"]:a["seg_start"] + a["seg_len"]] = False
    same = float((dx[single] == dxw[single]).float().mean())
    print("\n%s %s window %d: %d windows, dx rel-L2 %.3g, worst parameter %.3g (%s), "
          "single-crop samples bit-equal %.4f"
          % (cfg_name, precision, win, len(segs), rel_l2(dx, dxw), max(err.values()),
             max(err, key=err.get), same))
    assert set(grads) == set(gw)
    assert rel_l2(dx, dxw) < TOL[precision]
    assert max(err.values()) < TOL[precision]


@pytest.mark.parametrize("precision", ["fp32", "3xf16"])
def test_against_float64_oracle(precision):
    m = _model("cfg/frontend/PASE+.cfg", precision)
    L = 1_024_000 + 37
    x = seeded_randn((L,), 23, 0.5).cuda()
    win = enc.min_window(m.cfg)
    with torch.no_grad():
        cot = seeded_randn(tuple(m.extract_long(x, window=win).shape), 24).cuda()
    _, dx, grads = _long(m, x, cot, win)
    ref = {}
    for dt in (torch.float64, torch.float32):
        s = {k: (v.to(dt) if v.is_floating_point() else v) for k, v in m.state_dict().items()}
        leaves = {k: s[k].clone().requires_grad_(True) for k, _ in m.named_parameters()}
        s.update(leaves)
        xo = x.to(dt).view(1, 1, -1).requires_grad_(True)
        (O.encoder_forward(xo, s, m.cfg, training=False) * cot.to(dt)).sum().backward()
        ref[dt] = (xo.grad.view(-1), {k: v.grad for k, v in leaves.items()})
    dx64, p64 = ref[torch.float64]
    e32 = rel_l2(ref[torch.float32][0], dx64)
    perr = {k: rel_l2(grads[k], v) for k, v in p64.items() if float(v.norm()) > 0}
    print("\n%s: dx rel-L2 %.3g (float32 oracle %.3g), worst parameter %.3g (%s)"
          % (precision, rel_l2(dx, dx64), e32, max(perr.values()), max(perr, key=perr.get)))
    assert rel_l2(dx, dx64) < max(2 * e32, 2e-3)
    assert max(perr.values()) < 2e-3


def test_forty_million_samples():
    """A recording encode refuses (beyond its 32-bit indices): the backward completes in
    bounded memory, dx is finite, two windows agree and two runs are bit-identical."""
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    for _, p in m.named_parameters():
        p.requires_grad_(False)
    L = 40_000_000
    x = seeded_randn((L,), 29, 0.5).cuda()
    win = 1 << 20
    with torch.no_grad():
        T = m.extract_long(x, window=win).shape[-1]
    cot = seeded_randn((1, m.emb_dim, T), 30).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    _, dx1, _ = _long(m, x, cot, win)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    cap = enc.window_capacity(m.cfg, win)
    plans = m._grad_plan(cap, x.device).nbytes()
    # the bound of DESIGN.md section 20: the window's backward plan, plus O(L): the waveform's
    # clone and dx, four (emb, T') tensors (the output, y * cot, their gradients) and the state
    # log (the waveform, the cotangent and the forward's plan were allocated before the reset)
    bound = plans + 2 * 4 * L + 4 * 4 * m.emb_dim * T + 4 * 512 * (L // win + 2) + (256 << 20)
    print("\n40M samples: peak %.2f GB above the inputs, bound %.2f GB (backward plan %.2f GB)"
          % (peak / 1e9, bound / 1e9, plans / 1e9))
    assert peak <= bound
    assert bool(torch.isfinite(dx1).all())
    _, dx2, _ = _long(m, x, cot, win)
    assert torch.equal(dx1, dx2)
    _, dx3, _ = _long(m, x, cot, 1 << 19)
    print("windows 2^20 / 2^19: dx rel-L2 %.3g" % rel_l2(dx3, dx1))
    assert rel_l2(dx3, dx1) < 1e-5


def test_grad_sink_through_flat_adam():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    L = 400_000 + 37
    x = seeded_randn((L,), 31, 0.5).cuda()
    win = enc.min_window(m.cfg)
    with torch.no_grad():
        cot = seeded_randn(tuple(m.extract_long(x, window=win).shape), 32).cuda()
    _, dx, grads = _long(m, x, cot, win)
    from pase_b200.optim import FlatAdam
    opt = FlatAdam([p for _, p in m.named_parameters()], lr=1e-3).bind_encoder(m)
    opt.zero_grad(set_to_none=True)
    xl = x.clone().requires_grad_(True)
    (m.encode_long(xl, win) * cot).sum().backward()
    assert torch.equal(xl.grad, dx)
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, grads[k]), k
    m.grad_sink = None
