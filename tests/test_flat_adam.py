"""FlatAdam (one launch for all parameter groups) against torch.optim.Adam: the host logic
with the emulated kernel on CPU, and the CUDA kernel on the GPU."""
import copy

import pytest
import torch

import emul
import pase_b200.ops as ops
from pase_b200.optim import FlatAdam


def _nets(seed=0):
    torch.manual_seed(seed)
    a = torch.nn.Sequential(torch.nn.Linear(7, 13), torch.nn.PReLU(13), torch.nn.Linear(13, 5))
    return a, copy.deepcopy(a)


def _groups(net):
    # three groups with different hyper-parameters (frontend / two "workers"), odd sizes
    return [{"params": list(net[0].parameters()), "lr": 5e-3},
            {"params": list(net[1].parameters()), "lr": 1e-2, "weight_decay": 1e-2},
            {"params": list(net[2].parameters()), "lr": 2e-3, "betas": (0.8, 0.99), "eps": 1e-6}]


def _run(device, monkeypatch=None):
    ref, nat = _nets()
    ref, nat = ref.to(device), nat.to(device)
    o_ref = torch.optim.Adam(_groups(ref), lr=1e-3)
    o_nat = FlatAdam(_groups(nat), lr=1e-3)
    # parameters became views of ONE buffer, gradients of another
    assert all(p.data.untyped_storage().data_ptr() == o_nat.flat_param.untyped_storage().data_ptr()
               for p in nat.parameters())
    x = torch.randn(11, 7, device=device)
    for it in range(5):
        if it == 2:                       # an LR scheduler mutates param_groups in place
            for o in (o_ref, o_nat):
                o.param_groups[0]["lr"] = 1e-3
        for net, opt, none in ((ref, o_ref, True), (nat, o_nat, it % 2 == 0)):
            opt.zero_grad(set_to_none=none)          # both zero_grad conventions
            net(x).square().mean().backward()
            opt.step()
    for a, b in zip(ref.parameters(), nat.parameters()):
        assert torch.allclose(a, b, rtol=2e-5, atol=2e-7), float((a - b).abs().max())
    # state_dict in torch.optim.Adam's format: loads into a torch Adam and continues in step
    sd = o_nat.state_dict()
    ref2, _ = _nets()
    ref2 = ref2.to(device)
    ref2.load_state_dict(nat.state_dict())
    o_ref2 = torch.optim.Adam(_groups(ref2), lr=1e-3)
    o_ref2.load_state_dict(sd)
    # and back: a torch Adam state loads into a fresh FlatAdam
    _, nat2 = _nets()
    nat2 = nat2.to(device)
    nat2.load_state_dict(ref.state_dict())
    o_nat2 = FlatAdam(_groups(nat2), lr=1e-3)
    o_nat2.load_state_dict(o_ref.state_dict())
    for net, opt in ((ref2, o_ref2), (nat2, o_nat2), (ref, o_ref)):
        opt.zero_grad()
        net(x).square().mean().backward()
        opt.step()
    for a, b, c in zip(ref.parameters(), ref2.parameters(), nat2.parameters()):
        assert torch.allclose(a, b, rtol=2e-5, atol=2e-7) and torch.allclose(a, c, rtol=2e-5, atol=2e-7)
    return nat, o_nat, x


def test_flat_adam_matches_torch_adam_emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    nat, opt, x = _run("cpu")
    # facades: the reference scheduler's calling pattern (zero_grad per optimizer, backward,
    # step per optimizer) launches exactly once per iteration
    calls = []
    real = emul.call
    monkeypatch.setattr(ops, "call", lambda name, *a: (calls.append(name), real(name, *a))[1])
    views = opt.views()
    before = [p.detach().clone() for p in nat.parameters()]
    for v in views:
        v.zero_grad()
    nat(x).square().mean().backward()
    for v in views[:-1]:
        v.step()
    assert calls == []                                # deferred until the last group steps
    views[-1].step()
    assert calls == ["pase_adam_flat"]
    assert any(not torch.equal(a, b) for a, b in zip(before, nat.parameters()))
    sub = views[1].state_dict()
    assert len(sub["state"]) == 1 and sub["param_groups"][0]["lr"] == 1e-2


@pytest.mark.gpu
def test_flat_adam_matches_torch_adam_gpu():
    _run("cuda")
