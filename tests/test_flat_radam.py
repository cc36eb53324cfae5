"""RAdam groups in FlatAdam against the reference's own RAdam and Saver (tests/golden/radam.pt,
written by tests/golden/make_radam_golden.py): the golden trajectories with Adam and RAdam
groups in one engine, the state dict in the reference RAdam's format both ways, the per-group
facades and Saver files, and the algorithm check.  CPU, with the emulated kernel
(tests/emul/optim.py); tests/test_flat_radam_gpu.py runs the same checks on the CUDA kernel.

Tolerance (TOL, as for Adam in tests/test_flat_adam.py): the segment table holds lr and the
betas in fp32, where the reference uses Python floats.  The step size then differs by a few
1e-6 relatively (1 - fp32(0.999) is 1.3e-5 off 0.001, and the step size goes with its square
root), so over 12 steps of at most lr = 1e-2 a parameter moves at most ~1e-7 away from the
reference's, plus the fp32 rounding of its own ~1 magnitude.  DTOL bounds the displacement
from the initial value relatively, which a wrong step size of any group would exceed.
"""
import json
import os

import pytest
import torch

import emul
import pase_b200.ops as ops
from pase_b200 import Saver
from pase_b200.optim import FlatAdam

GOLD_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "radam.pt")
TOL = dict(rtol=2e-5, atol=2e-7)
DTOL = 2e-4
# the moments: exp_avg_sq is scaled by 1 - beta2, 1.3e-5 off for an fp32 0.999
MTOL = dict(rtol=2e-5, atol=1e-12)
ADAM_SHAPES = ((11, 3), (7,))
_GOLD = []


def gold():
    if not _GOLD:
        _GOLD.append(torch.load(GOLD_PATH, map_location="cpu", weights_only=False))
    return _GOLD[0]


def n_inst(gd):
    return sum(1 for k in gd if k.startswith("cfg/"))


def golden_params(gd, i, s):
    c = gd["cfg/%d" % i]
    key = "init/%d/%d" if s == 0 else "param/%d/%d/%%d" % (i, s)
    return [gd[key % (i, j) if s == 0 else key % j] for j in range(len(c["shapes"]))]


class Holder(torch.nn.Module):
    """The module a reference Saver wrapped for the golden files: parameters p0, p1, ..."""

    def __init__(self, params):
        super().__init__()
        for j, p in enumerate(params):
            self.register_parameter("p%d" % j, p)


def lr_at(gd, i, s):
    """The lr of instance i for step s (after the scheduler's change)."""
    meta = gd["meta"]
    lr = gd["cfg/%d" % i]["lr"]
    return lr * meta["lr_factor"] if s > meta["lr_change_after"] else lr


def setup(gd, device, at=0, seed=1):
    """An engine with an Adam group first (like --fe_opt Adam --min_opt radam) and one RAdam
    group per golden instance, its parameters at golden step `at`; and a torch Adam over a
    copy of the Adam group."""
    g0 = torch.Generator().manual_seed(seed)
    init = [torch.randn(s, generator=g0) for s in ADAM_SHAPES]
    adam_p = [torch.nn.Parameter(t.clone().to(device)) for t in init]
    ref_p = [torch.nn.Parameter(t.clone().to(device)) for t in init]
    groups = [{"params": adam_p, "lr": 3e-3, "weight_decay": 1e-2, "algorithm": "adam"}]
    for i in range(n_inst(gd)):
        c = gd["cfg/%d" % i]
        groups.append({"params": [torch.nn.Parameter(t.clone().to(device))
                                  for t in golden_params(gd, i, at)],
                       "lr": lr_at(gd, i, at + 1), "betas": c["betas"],
                       "weight_decay": c["weight_decay"]})
    engine = FlatAdam(groups, algorithm="radam")
    ref = torch.optim.Adam(ref_p, lr=3e-3, weight_decay=1e-2)
    return engine, ref


def feed(engine, ref, gd, s, seed=1):
    """Step s's gradients: the golden ones for the RAdam groups, seeded ones for Adam."""
    gen = torch.Generator().manual_seed(1000 * seed + s)
    for j, a in enumerate(engine.param_groups[0]["params"]):
        a.grad = torch.randn(a.shape, generator=gen).to(a.device)
        if ref is not None:
            ref.param_groups[0]["params"][j].grad = a.grad.clone()
    for i, grp in enumerate(engine.param_groups[1:]):
        for j, p in enumerate(grp["params"]):
            p.grad = gd["grad/%d/%d/%d" % (i, s, j)].to(p.device)


def step(engine, ref, gd, s, seed=1):
    """Golden step s: the scheduler's lr change, the gradients, one launch, torch Adam."""
    if s == gd["meta"]["lr_change_after"] + 1:
        for grp in engine.param_groups[1:]:
            grp["lr"] *= gd["meta"]["lr_factor"]
    feed(engine, ref, gd, s, seed)
    engine.step()
    if ref is not None:
        ref.step()


def check(engine, ref, gd, s, tol=TOL):
    for i, grp in enumerate(engine.param_groups[1:]):
        for j, (p, want) in enumerate(zip(grp["params"], golden_params(gd, i, s))):
            got = p.detach().cpu()
            assert torch.allclose(got, want, **tol), (s, i, j, float((got - want).abs().max()))
            d_got, d_want = got - golden_params(gd, i, 0)[j], want - golden_params(gd, i, 0)[j]
            err = float((d_got - d_want).abs().max() / d_want.abs().max())
            assert err < DTOL, (s, i, j, err)
    if ref is not None:
        for a, b in zip(engine.param_groups[0]["params"], ref.param_groups[0]["params"]):
            assert torch.allclose(a, b, **tol), (s, float((a - b).abs().max()))


def run_golden(device):
    gd = gold()
    engine, ref = setup(gd, device)
    for s in range(1, gd["meta"]["steps"] + 1):
        step(engine, ref, gd, s)
        check(engine, ref, gd, s)
    return engine


def state_roundtrip(device):
    """At step 8: the engine's RAdam groups' state is the golden state in the reference's
    format; a fresh engine loaded from the engine's state continues bit for bit; one loaded
    from the golden state (through the facades) follows the golden trajectory."""
    gd = gold()
    engine, ref = setup(gd, device)
    for s in range(1, 9):
        step(engine, ref, gd, s)
    full = engine.state_dict()
    views = engine.views()
    for i in range(n_inst(gd)):
        want, got = gd["state8/%d" % i], views[i + 1].state_dict()
        assert got["param_groups"] == want["param_groups"], (got["param_groups"], want)
        assert sorted(got["state"]) == sorted(want["state"])
        for k, st in want["state"].items():
            assert type(got["state"][k]["step"]) is int and got["state"][k]["step"] == st["step"]
            for name in ("exp_avg", "exp_avg_sq"):
                assert torch.allclose(got["state"][k][name].cpu(), st[name], **MTOL), name
    # the Adam group stays in torch.optim.Adam's format
    assert "amsgrad" in full["param_groups"][0] and "algorithm" not in full["param_groups"][0]
    assert torch.is_tensor(full["state"][0]["step"])
    # engine -> fresh engine (full dict) and golden -> fresh engine (one facade per instance)
    e_own, _ = setup(gd, device)
    for a, b in zip(e_own._plist, engine._plist):
        a.data.copy_(b.data)
    e_own.load_state_dict(full)
    e_gold, _ = setup(gd, device, at=8)
    for a, b in zip(e_gold.param_groups[0]["params"], engine.param_groups[0]["params"]):
        a.data.copy_(b.data)
    e_gold.views()[0].load_state_dict(views[0].state_dict())
    for i, v in enumerate(e_gold.views()[1:]):
        v.load_state_dict(gd["state8/%d" % i])
    for e in (e_own, e_gold):
        assert [g["lr"] for g in e.param_groups] == [g["lr"] for g in engine.param_groups]
    for s in range(9, gd["meta"]["steps"] + 1):
        step(engine, ref, gd, s)
        step(e_own, None, gd, s)
        step(e_gold, None, gd, s)
        for name in ("flat_param", "exp_avg", "exp_avg_sq", "steps"):
            assert torch.equal(getattr(engine, name), getattr(e_own, name)), (s, name)
        check(e_gold, ref, gd, s)
        check(engine, ref, gd, s)


def _dump(d, files):
    os.makedirs(d, exist_ok=True)
    for name, t in files.items():
        with open(os.path.join(d, name), "wb") as f:
            f.write(bytes(t.tolist()))
    return d


def saver_interchange(device, tmp_path):
    """The reference Saver's files load through a facade and continue on the golden
    trajectory; the native Saver around a facade writes the same index and checkpoints."""
    gd = gold()
    meta = gd["meta"]
    k = meta["saver_instance"]
    files = {n[len("saver/file/"):]: v for n, v in gd.items() if n.startswith("saver/file/")}
    index = json.loads(bytes(files["M-radam-checkpoints"].tolist()).decode())
    last = max(meta["saver_steps"])
    # reference writes, native reads: the latest checkpoint is step `last`
    engine, ref = setup(gd, device, at=last)
    view = engine.views()[k + 1]
    holder = Holder(engine.param_groups[k + 1]["params"])
    for p in holder.parameters():
        p.data.zero_()
    saver = Saver(holder, _dump(str(tmp_path / "ref"), files), optimizer=view, prefix="M-radam-")
    assert saver.load_weights() is True
    for p, want in zip(holder.parameters(), golden_params(gd, k, last)):
        assert torch.equal(p.detach().cpu(), want)
    assert float(engine.steps[k + 1]) == last
    for s in range(last + 1, meta["steps"] + 1):
        step(engine, None, gd, s)
        for p, want in zip(engine.param_groups[k + 1]["params"], golden_params(gd, k, s)):
            assert torch.allclose(p.detach().cpu(), want, **TOL), s
    # native writes the same sequence
    engine, ref = setup(gd, device)
    view = engine.views()[k + 1]
    holder = Holder(engine.param_groups[k + 1]["params"])
    d = str(tmp_path / "native")
    saver = Saver(holder, d, optimizer=view, prefix="M-radam-")
    for s in range(1, last + 1):
        step(engine, ref, gd, s)
        if s in meta["saver_steps"]:
            saver.save("W", s)
    assert sorted(os.listdir(d)) == sorted(files)
    assert json.load(open(os.path.join(d, "M-radam-checkpoints"))) == index
    for name in files:
        if not name.startswith("weights_"):
            continue
        want = torch.load(os.path.join(tmp_path / "ref", name), map_location="cpu",
                          weights_only=False)
        got = torch.load(os.path.join(d, name), map_location="cpu", weights_only=False)
        assert list(got) == list(want) and got["step"] == want["step"]
        assert list(got["state_dict"]) == list(want["state_dict"])
        for key, v in want["state_dict"].items():
            assert torch.allclose(got["state_dict"][key], v, **TOL), key
        go, wo = got["optimizer"], want["optimizer"]
        assert go["param_groups"] == wo["param_groups"]
        assert sorted(go["state"]) == sorted(wo["state"])
        for i, st in wo["state"].items():
            assert type(go["state"][i]["step"]) is int and go["state"][i]["step"] == st["step"]
            for n in ("exp_avg", "exp_avg_sq"):
                assert torch.allclose(go["state"][i][n], st[n], **MTOL), n


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)


def test_golden_trajectories_mixed_engine_emulated(emulated):
    engine = run_golden("cpu")
    assert [g["algorithm"] for g in engine.param_groups] == ["adam"] + ["radam"] * n_inst(gold())


def test_state_dict_both_ways_emulated(emulated):
    state_roundtrip("cpu")


def test_facades_and_saver_interchange_emulated(emulated, tmp_path):
    saver_interchange("cpu", tmp_path)


def test_algorithm_in_segment_table_emulated(emulated):
    """The table's algorithm column follows the groups, and a change rewrites the table."""
    import struct
    gd = gold()
    engine, _ = setup(gd, "cpu")
    codes = lambda: [struct.unpack_from(emul.optim.ROW, engine._segments().numpy().tobytes(),
                                        48 * i)[7] for i in range(len(engine.param_groups))]
    assert codes() == [0.0] + [1.0] * n_inst(gd)
    engine.param_groups[1]["algorithm"] = "adam"
    assert codes() == [0.0, 0.0] + [1.0] * (n_inst(gd) - 1)


def test_unknown_algorithm_raises():
    p = [torch.nn.Parameter(torch.zeros(3))]
    with pytest.raises(ValueError, match="algorithm"):
        FlatAdam(p, algorithm="adamw")
    with pytest.raises(ValueError, match="algorithm"):
        FlatAdam([{"params": p, "algorithm": "sgd"}])
    engine = FlatAdam([{"params": p, "algorithm": "RAdam".lower()}])
    engine.param_groups[0]["algorithm"] = "plainradam"
    with pytest.raises(ValueError, match="algorithm"):
        engine._segments()
