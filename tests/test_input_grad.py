"""The waveform gradient of WaveFe (DESIGN.md section 17) on the CPU with emulated kernels
(tests/emul/): the host-side routing, the sinc layer's haloed / banded polyphase
GEMM formulation and the reflect fold-back against float64 autograd through the oracle, and the
launches of the data-gradient-only sweep of a frozen encoder."""
import pytest
import torch

import emul
import pase_oracle as O
from helpers import load_golden, resolve_cfg, fill_state_dict, seeded_randn, rel_l2
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import WaveFe


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    yield


CONFIGS = {"pasep": "enc_pasep_train_3200", "pase": "enc_pase_train_2400",
           "mini": "enc_mini_train_1763", "mininornn": "enc_mininornn_train_1600"}


def make_model(key, precision, training, frozen=False):
    gold, meta = load_golden(CONFIGS[key])
    cfg = resolve_cfg(meta["cfg"])
    model = WaveFe(**cfg)
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), meta["seed"]))
    model.train(training)
    if frozen:
        model.requires_grad_(False)
    return model, cfg, meta


class Ref(object):
    """dL/dx of L = sum(y * cot) through the oracle with the model's parameters: `dx` in
    float64, `tol` = max(1e-4, 2 x the float32 oracle's own relative L2 error).  The float32
    term matters where a PReLU input sits within float32 rounding of its kink: the PASE.cfg
    train case has one in the sinc layer, and there the float32 oracle itself is 1.2e-3 off."""

    def __init__(self, model, cfg, x, cot, training):
        sd = model.state_dict()
        out = []
        for dt in (torch.float64, torch.float32):
            s = {k: (v.to(dt) if v.is_floating_point() else v) for k, v in sd.items()}
            xx = x.detach().to(dt).requires_grad_(True)
            y = O.encoder_forward(xx, s, cfg, training=training)
            (y * cot.to(dt)).sum().backward()
            out.append(xx.grad)
        self.dx = out[0]
        self.tol = max(1e-4, 2 * rel_l2(out[1], out[0]))


def oracle_dx(model, cfg, x, cot, training):
    return Ref(model, cfg, x, cot, training)


def native_dx(model, x, cot):
    x = x.detach().clone().requires_grad_(True)
    y, _ = model._encode(x)
    (y * cot).sum().backward()
    return y, x.grad


def check_dx(got, ref, edge=300):
    tol, ref = ref.tol, ref.dx
    assert got is not None and got.shape == ref.shape and got.dtype == torch.float32
    assert rel_l2(got, ref) < tol, rel_l2(got, ref)
    # the first and last samples of every recording: a reflect fold-back or a sample boundary
    # gone wrong shows there first
    for sl in (slice(0, edge), slice(-edge, None)):
        assert rel_l2(got[..., sl], ref[..., sl]) < tol, (sl, rel_l2(got[..., sl], ref[..., sl]))


@pytest.mark.parametrize("precision", ["fp32", "3xtf32"])
@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("key", list(CONFIGS))
def test_dx_matches_float64_oracle(key, training, precision, emulated):
    """fold 4 (fp32) and fold 32 (3xtf32) plans, train- and eval-mode BatchNorm."""
    model, cfg, meta = make_model(key, precision, training)
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        y, _ = model._encode(x)
    model.load_state_dict(state)            # the oracle sees the running statistics used
    cot = seeded_randn(tuple(y.shape), meta["seed"] + 2)
    _, dx = native_dx(model, x, cot)
    model.load_state_dict(state)
    check_dx(dx, oracle_dx(model, cfg, x, cot, training))


@pytest.mark.parametrize("precision", ["fp32", "3xtf32"])
@pytest.mark.parametrize("case", ["min_length", "odd_length", "single", "distinct"])
def test_dx_edges(case, precision, emulated):
    """The encoder's minimum length, a length that is no multiple of the fold, N = 1, and a
    batch whose recordings differ (eval mode: each one's dx must be its own, so dy frames
    leaking across a sample boundary show)."""
    training = case != "distinct"
    model, cfg, meta = make_model("mini", precision, training, frozen=case == "distinct")
    N, T = 2, 1763
    if case == "min_length":
        T = enc.min_length(model.cfg)
    elif case == "odd_length":
        T = 1763 + 2 * 32 + 1            # T mod 32 = 10, T mod 4 = 2
    elif case == "single":
        N = 1
    x = seeded_randn((N, 1, T), 11, 0.5)
    if case == "distinct":
        x = torch.cat([x[:1], 3.0 * seeded_randn((1, 1, T), 12, 1.0)])
    with torch.no_grad():
        y, _ = model._encode(x)
    cot = seeded_randn(tuple(y.shape), 13)
    _, dx = native_dx(model, x, cot)
    ref = oracle_dx(model, cfg, x, cot, training)
    check_dx(dx, ref, edge=min(300, T))
    if case == "distinct":
        for n in range(N):       # the same recording alone
            _, dx1 = native_dx(model, x[n:n + 1], cot[n:n + 1])
            assert rel_l2(dx1, ref.dx[n:n + 1]) < ref.tol
            assert rel_l2(dx[n:n + 1], dx1) < 1e-6


def _record(monkeypatch, plan_of):
    """Wrap ops.call: (name, args) with plan-owned tensors as their address and other tensors
    as (dtype, numel)."""
    seen = []

    def norm(a, owned):
        if isinstance(a, torch.Tensor):
            return ("plan", a.data_ptr()) if a.untyped_storage().data_ptr() in owned else \
                ("tmp", str(a.dtype), a.numel())
        return a

    def spy(name, *args):
        plan = plan_of()
        owned = {t.untyped_storage().data_ptr() for t in plan.tensors()} if plan else set()
        seen.append((name, tuple(norm(a, owned) for a in args)))
        return emul.call(name, *args)
    monkeypatch.setattr(ops, "call", spy)
    return seen


def _step(model, x, cot):
    model.zero_grad(set_to_none=True)
    y, _ = model._encode(x)
    (y * cot).sum().backward()
    return y.detach(), {k: p.grad for k, p in model.named_parameters()}


@pytest.mark.parametrize("precision", ["fp32", "3xf16"])
def test_launches_unchanged_without_input_grad(precision, monkeypatch):
    """x without requires_grad: exactly the forward and sweep the encoder ran before it could
    return dx (_EncoderFn forward + encoder_backward with no dx), argument for argument, and no
    input-gradient buffer; with x.requires_grad the outputs and every parameter gradient are
    bit-equal and dx is returned on top."""
    model, cfg, meta = make_model("pasep", precision, True)
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    plan_of = lambda: model._plans.get((meta["N"], meta["T"], "cpu", precision))
    seen = _record(monkeypatch, plan_of)
    with torch.no_grad():
        y0, _ = model._encode(x)
    cot = seeded_randn(tuple(y0.shape), meta["seed"] + 2)
    _step(model, x, cot)                        # warm-up: the plan and its operand buffers
    plan = plan_of()
    assert plan.dyh is None and plan.dxpad[0] is None

    # the sweep as the encoder ran it before the input gradient existed
    named = list(model.named_parameters())
    params = dict(named)
    del seen[:]
    model.zero_grad(set_to_none=True)
    out, out_ntc = enc.encoder_forward(plan, model, x, params, True, True)
    # autograd materialises the unused second output's gradient as zeros
    enc.encoder_backward(plan, model, params, cot.contiguous(), torch.zeros_like(out_ntc), True,
                         None)
    before = list(seen)

    del seen[:]
    y1, g1 = _step(model, x, cot)
    assert seen == before
    assert plan.dyh is None and plan.dxpad[0] is None

    xr = x.clone().requires_grad_(True)
    del seen[:]
    model.zero_grad(set_to_none=True)
    y2, _ = model._encode(xr)
    (y2 * cot).sum().backward()
    g2 = {k: p.grad for k, p in model.named_parameters()}
    assert torch.equal(y1, y2.detach())
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    assert xr.grad is not None and xr.grad.shape == x.shape
    names = [n for n, _ in seen]
    assert names.count("pase_reflect_fold_wave") == 1 and names.count("pase_sinc_dgrad_pack") == 1


@pytest.mark.parametrize("training", [True, False])
def test_frozen_encoder_runs_the_data_gradient_sweep_only(training, monkeypatch):
    """A frozen encoder: no weight-gradient GEMM, pase_sinc_grad, colsum, weight re-layout back,
    cast or scatter; the BatchNorm/PReLU reductions still run once per block; dx is bit-equal
    to the full sweep's; no parameter gets a .grad."""
    model, cfg, meta = make_model("pasep", "3xf16", training)
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    plan_of = lambda: model._plans.get((meta["N"], meta["T"], "cpu", "3xf16"))
    seen = _record(monkeypatch, plan_of)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        y0, _ = model._encode(x)
    cot = seeded_randn(tuple(y0.shape), meta["seed"] + 2)

    model.load_state_dict(state)
    _, dx_full = native_dx(model, x, cot)

    model.load_state_dict(state)
    model.requires_grad_(False)
    del seen[:]
    y, dx = native_dx(model, x, cot)
    names = [n for n, _ in seen]
    banned = ("pase_gemm_tn", "pase_tc_gemm_tn", "pase_sinc_grad", "pase_colsum",
              "pase_scatter_copy", "pase_cast_d2f")
    assert not [n for n in names if n.startswith(banned)], names
    assert [a[3] for n, a in seen if n == "pase_conv_w_batch"] in ([0, 1], [3, 4])
    nblk = len(cfg["kwidths"])
    assert names.count("pase_bn_prelu_bwd_reduce") == nblk
    assert names.count("pase_bn_prelu_bwd_apply_src") == nblk
    assert all(p.grad is None for p in model.parameters())
    assert torch.equal(dx, dx_full)
    check_dx(dx, oracle_dx(model, cfg, x, cot, training))


def test_frozen_encoder_without_input_grad_stays_forward_only(emulated):
    """Nothing needs a gradient: the forward alone, no backward buffers, a detached output."""
    model, cfg, meta = make_model("pasep", "3xf16", False, frozen=True)
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    y, _ = model._encode(x)
    plan = model._plan(meta["N"], meta["T"], x.device)
    assert not y.requires_grad and not plan.backward_ready and plan.dyz is None


def test_grad_sink_with_input_grad(emulated):
    """FlatAdam.bind_encoder: the parameter gradients still go to the flat buffer, bit-equal to
    a run whose input needs no gradient, and dx is returned."""
    from pase_b200.optim import FlatAdam
    model, cfg, meta = make_model("pasep", "3xf16", True)
    opt = FlatAdam(list(model.parameters()), lr=1e-3).bind_encoder(model)
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        y0, _ = model._encode(x)
    cot = seeded_randn(tuple(y0.shape), meta["seed"] + 2)
    model.load_state_dict(state)
    opt.zero_grad(set_to_none=True)
    y, _ = model._encode(x)
    (y * cot).sum().backward()
    g1 = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.load_state_dict(state)
    opt.zero_grad(set_to_none=True)
    y, dx = native_dx(model, x, cot)
    for k, p in model.named_parameters():
        assert torch.equal(p.grad, g1[k]), k
    check_dx(dx, oracle_dx(model, cfg, x, cot, True))
