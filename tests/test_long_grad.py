"""WaveFe.encode_long (DESIGN.md section 20) on the CPU with emulated kernels
(tests/emul/): features, waveform and parameter gradients of recordings of three
or more windows against float64 autograd through the oracle, a cotangent on one crop, short
recordings against encode_packed, the frozen sweep, grad_sink, the plan-generation guard shared
with encode_packed, and the refusals, all raised before any launch."""
import pytest
import torch

import emul
import pase_oracle as O
from helpers import load_golden, resolve_cfg, fill_state_dict, seeded_randn, rel_l2
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import WaveFe

CPU = torch.device("cpu")
CONFIGS = ["cfg/frontend/PASE+.cfg", "cfg/frontend/PASE.cfg", "mini", "mininornn"]
MINI = {"mini": "enc_mini_train_1763", "mininornn": "enc_mininornn_train_1600"}


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    yield


def make_model(cfg_name, precision="fp32", seed=11):
    cfg = load_golden(MINI[cfg_name])[1]["cfg"] if cfg_name in MINI else cfg_name
    model = WaveFe(**resolve_cfg(cfg))
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    return model.eval()


def freeze(model, frozen=True):
    for p in model.parameters():
        p.requires_grad_(not frozen)


def long_length(model):
    """Three windows at the minimum window: two full ones and a shorter last one."""
    w = enc.min_window(model.cfg)
    L = 2 * w + 40037
    assert len(enc.plan_windows(model.cfg, L, w)) >= 3
    return L, w


def run_long(model, x, cot, window):
    """encode_long + backward of <y, cot> -> (y, dx, {name: grad})."""
    x = x.detach().clone().requires_grad_(True)
    for _, p in model.named_parameters():        # Model.parameters() skips frozen ones
        p.grad = None
    y = model._encode_long(x, window, CPU)
    (y * cot).sum().backward()
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    return y, x.grad, grads


def oracle(model, w, cot, dtype):
    """Autograd through the oracle in `dtype`: features, dx and parameter gradients of <y, cot>
    for the whole recording."""
    s = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    leaves = {k: s[k].clone().requires_grad_(True) for k, _ in model.named_parameters()}
    s.update(leaves)
    x = w.to(dtype).view(1, 1, -1).requires_grad_(True)
    y = O.encoder_forward(x, s, model.cfg, training=False)
    (y * cot.to(dtype)).sum().backward()
    return y.detach(), x.grad.view(-1), {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("name", CONFIGS)
def test_matches_float64_oracle(name, emulated):
    model = make_model(name)
    L, w = long_length(model)
    x = seeded_randn((L,), 300 + len(name), 0.5)
    with torch.no_grad():
        feats = model._extract_long(x, None, w, CPU)
    cot = seeded_randn(tuple(feats.shape), 31)
    y, dx, grads = run_long(model, x, cot, w)
    assert torch.equal(y, feats)
    y64, dx64, p64 = oracle(model, x, cot, torch.float64)
    y32, dx32, p32 = oracle(model, x, cot, torch.float32)
    tol = lambda a, b: max(1e-4, 2 * rel_l2(a, b))
    assert rel_l2(y, y64) < tol(y32, y64)
    assert rel_l2(dx, dx64) < tol(dx32, dx64), (rel_l2(dx, dx64), rel_l2(dx32, dx64))
    assert set(grads) == set(p64)
    for k, v in p64.items():
        if float(v.norm()) == 0.0:
            continue
        assert rel_l2(grads[k], v) < tol(p32[k], v), (k, rel_l2(grads[k], v), rel_l2(p32[k], v))


@pytest.mark.parametrize("name", ["cfg/frontend/PASE.cfg", "mini"])
def test_single_crop_cotangent(name, emulated):
    """A cotangent on the middle window's crop only: dx is zero past the crop's receptive field
    (before it too without a QRNN, whose state reaches back to the first sample), equals the
    whole-recording packed backward's up to summation order, and matches the oracle with the
    whole-recording backward's own error (mini: a few samples near a PReLU kink put both at
    7e-4, against 5e-7 for the float32 oracle)."""
    model = make_model(name)
    freeze(model)
    L, w = long_length(model)
    cfg, hop = model.cfg, enc.hop_size(model.cfg)
    segs = enc.plan_windows(cfg, L, w)
    s = segs[1]
    f0 = s["seg_start"] // hop + s["crop_f0"]
    f1 = f0 + s["crop_n"]
    x = seeded_randn((L,), 41, 0.5)
    T = enc.frame_counts(cfg, L)[-1]
    cot = torch.zeros(1, model.emb_dim, T)
    cot[..., f0:f1] = seeded_randn((1, model.emb_dim, f1 - f0), 42)
    _, dx, _ = run_long(model, x, cot, w)
    A, B = enc.receptive_field(cfg)
    assert float(dx[hop * (f1 - 1) + B + 1:].abs().max()) == 0.0
    if not cfg["rnn_pool"]:
        assert float(dx[:hop * f0 - A].abs().max()) == 0.0
    xp = x.clone().requires_grad_(True)
    (model._encode_packed([xp], L, CPU)[0] * cot).sum().backward()
    assert rel_l2(dx, xp.grad) < 1e-6
    _, dx64, _ = oracle(model, x, cot, torch.float64)
    _, dx32, _ = oracle(model, x, cot, torch.float32)
    assert rel_l2(dx, dx64) < max(2e-3, 2 * rel_l2(dx32, dx64), 2 * rel_l2(xp.grad, dx64))


def test_short_recording_is_encode_packed(emulated):
    model = make_model("mini")
    w = enc.min_window(model.cfg)
    x = seeded_randn((w - 777,), 5, 0.5)
    with torch.no_grad():
        cot = seeded_randn(tuple(model._encode_packed([x], w, CPU)[0].shape), 6)
    y, dx, grads = run_long(model, x, cot, w)
    xp = x.clone().requires_grad_(True)
    model.zero_grad(set_to_none=True)
    yp = model._encode_packed([xp], w, CPU)[0]
    assert type(y.grad_fn) is type(yp.grad_fn)
    (yp * cot).sum().backward()
    assert torch.equal(y, yp) and torch.equal(dx, xp.grad)
    for k, p in model.named_parameters():
        assert torch.equal(grads[k], p.grad), k


def test_frozen_sweep(emulated, monkeypatch):
    """All parameters frozen: the data-gradient sweep (no weight-gradient GEMM, no parameter
    gradient) gives the full sweep's dx."""
    model = make_model("cfg/frontend/PASE+.cfg")
    L, w = long_length(model)
    x = seeded_randn((L,), 51, 0.5)
    with torch.no_grad():
        cot = seeded_randn(tuple(model._extract_long(x, None, w, CPU).shape), 52)
    _, dx_full, grads = run_long(model, x, cot, w)
    assert grads
    freeze(model)
    names = []
    monkeypatch.setattr(ops, "call",
                        lambda n, *a: (names.append(n), emul.call(n, *a))[1])
    _, dx, grads = run_long(model, x, cot, w)
    assert torch.equal(dx, dx_full) and not grads
    assert "pase_sinc_grad" not in names and "pase_axpy" not in names
    assert "pase_qrnn_scan_bwd_carry_var" in names


def test_grad_sink_equals_autograd(emulated):
    model = make_model("mini")
    L, w = long_length(model)
    x = seeded_randn((L,), 61, 0.5)
    with torch.no_grad():
        cot = seeded_randn(tuple(model._extract_long(x, None, w, CPU).shape), 62)
    _, dx, grads = run_long(model, x, cot, w)
    sink = {k: torch.full_like(p, float("nan")) for k, p in model.named_parameters()}
    model.grad_sink = sink
    _, dx2, grads2 = run_long(model, x, cot, w)
    assert torch.equal(dx, dx2) and not grads2
    for k, v in grads.items():
        assert torch.equal(sink[k], v), k


def test_backward_bumps_the_shared_plan_generation(emulated):
    """encode_long's backward recomputes on the encode_packed plan of window_capacity samples:
    a pending encode_packed backward on that plan raises afterwards."""
    model = make_model("mini")
    L, w = long_length(model)
    cap = enc.window_capacity(model.cfg, w)
    xp = seeded_randn((3000,), 71, 0.5).requires_grad_(True)
    yp = model._encode_packed([xp], cap, CPU)[0]
    x = seeded_randn((L,), 72, 0.5).requires_grad_(True)
    model._encode_long(x, w, CPU).sum().backward()
    assert x.grad is not None
    with pytest.raises(RuntimeError, match="overwritten"):
        yp.sum().backward()


def test_refusals_before_any_launch(emulated):
    model = make_model("cfg/frontend/PASE+.cfg")
    cfg = model.cfg
    L, w = long_length(model)
    n0 = ops.launch_count
    x = torch.zeros(L)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.encode_long(x)                                    # a CPU module
    with pytest.raises(RuntimeError, match="device"):
        model._encode_long(x, w, torch.device("cuda"))           # a waveform elsewhere
    with pytest.raises(ValueError, match="window"):
        model._encode_long(x, w - 160, CPU)
    with pytest.raises(ValueError, match="shorter"):
        model._encode_long(torch.zeros(enc.min_length(cfg) - 1), w, CPU)
    bad = 2 * w + 160 * 300 + 155                               # L mod 160 in 151..159
    with pytest.raises(NotImplementedError, match="pools its dense skips"):
        model._encode_long(torch.zeros(bad), w, CPU)
    with pytest.raises(TypeError):
        model._encode_long(torch.zeros(L, dtype=torch.float64), w, CPU)
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        model.encode_long(x)
    assert ops.launch_count == n0


def test_in_place_update_refused_before_any_launch(emulated):
    model = make_model("mini")
    L, w = long_length(model)
    x = seeded_randn((L,), 81, 0.5).requires_grad_(True)
    y = model._encode_long(x, w, CPU)
    with torch.no_grad():
        model.W.weight.add_(0.01)
    n0 = ops.launch_count
    with pytest.raises(RuntimeError, match="inplace"):
        y.sum().backward()
    assert ops.launch_count == n0 and x.grad is None
