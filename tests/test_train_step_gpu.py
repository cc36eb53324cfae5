"""The captured PASE/PASE+ training step on the GPU: GraphedTrainStep equals the eager loop
(batcher -> model -> total_loss -> backward -> FlatAdam.step) bit for bit over warm-up, capture
and replays, with every call issued without a synchronise and an lr schedule changing every
group before every call; FlatAdam's table follows lr changes under GraphedEncoderStep; the SPC
gather kernels equal the torch gather they replace; a replayed step launches nothing from
Python and copies one plan in and one loss vector out.
"""
import os
import random

import numpy as np
import pytest
import torch

from distortion_banks import build_banks, case_cfg
from helpers import fill_state_dict, resolve_cfg, seeded_randn
from pase_b200 import _lib, ops
from pase_b200 import functional as Fn
from pase_b200.batch import DeviceBatcher, WavPool
from pase_b200.distortions import config_distortions
from pase_b200.graph import GraphedEncoderStep, GraphedTrainStep
from pase_b200.optim import FlatAdam
from pase_b200.pase import total_loss
from test_train_step import (RECIPES, SPC_CASES, _frames, build_corpus, check_strided_rows,
                             make_model, spc_reference)

pytestmark = pytest.mark.gpu

HOP = 160


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("train_step_gpu"))
    data_root, cfg = build_corpus(root, 40, 32001, 64000)
    return dict(root=root, data_root=data_root, cfg=cfg,
                banks=build_banks(os.path.join(root, "banks")))


def _setup(corpus, recipe, T, precision, seed=5):
    fe, wcfg, _ = RECIPES[recipe]
    model = make_model(recipe)
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    model.frontend.precision = precision
    model = model.cuda().train()
    # one group per module, like the reference trainer's optimizers
    groups = [{"params": list(model.frontend.parameters())}]
    groups += [{"params": list(w.parameters())} for w in
               list(model.classification_workers) + list(model.regression_workers)]
    engine = FlatAdam(groups, lr=5e-4).bind_encoder(model.frontend)
    wavs = WavPool(corpus["data_root"], corpus["cfg"], "train", placement="cuda")
    dist = None
    if recipe == "pase+":
        dist = config_distortions(device="cuda", **case_cfg("pase_plus", corpus["banks"])[0])
    batcher = DeviceBatcher.from_train_opts(
        wcfg, T, HOP, wavs, random_scale=True, distortions=dist,
        trans_cache=os.path.join(corpus["root"], "cache_" + recipe))
    return model, engine, batcher


def _batches(n, B, steps, seed):
    """Index lists of `steps` batches, epoch by epoch (True marks an epoch's first batch)."""
    rng = np.random.RandomState(seed)
    out = []
    while len(out) < steps:
        perm = rng.permutation(n).tolist()
        for j in range(0, n - B + 1, B):
            out.append((j == 0, perm[j:j + B]))
    return out[:steps]


def _poly(engine, k, steps):
    for gi, g in enumerate(engine.param_groups):
        g["lr"] = (5e-4 + 1e-5 * gi) * (1.0 - k / (steps + 1.0)) ** 0.9


def _seed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def _triple(s):
    return (random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def _compare(ea, ga):
    for name, a, b in (("flat_param", ea.flat_param, ga.flat_param),
                       ("exp_avg", ea.exp_avg, ga.exp_avg),
                       ("exp_avg_sq", ea.exp_avg_sq, ga.exp_avg_sq), ("steps", ea.steps, ga.steps)):
        assert torch.equal(a, b), name


CASES = [("pase+", "3xf16", 4, 16000, False), ("pase+", "bf16", 4, 16000, False),
         ("pase+", "3xf16", 32, 32000, False), ("pase", "3xf16", 4, 16000, False),
         ("pase", "fp32", 4, 16000, True)]


@pytest.mark.parametrize("recipe,precision,B,T,triple", CASES)
def test_graphed_steps_equal_the_eager_loop(recipe, precision, B, T, triple, corpus):
    steps = 6
    prev = Fn.PRECISION
    Fn.set_precision(precision)
    try:
        batches = _batches(len(WavPool(corpus["data_root"], corpus["cfg"], "train",
                                       placement="cpu")), B, steps, 11)
        # eager: the public path, the generators seeded globally (SPC draws from `random`)
        model, engine, batcher = _setup(corpus, recipe, T, precision)
        _seed(3)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                batcher.reset()
            _poly(engine, k, steps)
            engine.zero_grad(set_to_none=True)
            batch = batcher(idx)
            _, _, preds, labels = model(batch)
            tot, losses = total_loss(model, preds, labels)
            tot.backward()
            engine.step()
        eager = dict({n: float(v.detach()) for n, v in losses.items()}, total=float(tot.detach()))
        torch.cuda.synchronize()
        # graphed: the same draws, every call issued without a synchronise
        gmodel, gengine, gbatcher = _setup(corpus, recipe, T, precision)
        step = GraphedTrainStep(gmodel, gengine, gbatcher, B)
        rng = None
        if triple:
            rng = _triple(3)
        else:
            _seed(3)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                gbatcher.reset()
            _poly(gengine, k, steps)
            step(idx, rng)
        assert step.graph is not None and step.calls == steps
        got = step.losses()
        torch.cuda.synchronize()
        assert set(got) == set(eager)
        for n in eager:
            assert got[n] == eager[n], (n, got[n], eager[n])
        _compare(engine, gengine)
        if recipe == "pase":
            assert len(step.planner.spc) == 1
    finally:
        Fn.set_precision(prev)


def test_replay_launches_and_copies(corpus):
    B, T = 4, 16000
    model, engine, batcher = _setup(corpus, "pase", T, "3xf16")
    step = GraphedTrainStep(model, engine, batcher, B, warmup=1)
    batches = _batches(len(batcher.wavs), B, 4, 2)
    for _, idx in batches[:2]:                   # warm-up, capture + replay
        step(idx)
    with pytest.raises(ValueError, match="batch of 3"):
        step(batches[2][1][:3])
    torch.cuda.synchronize()
    n0 = ops.launch_count
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step(batches[2][1])
        torch.cuda.synchronize()
    assert ops.launch_count == n0
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    h2d = [n for n in names if "HtoD" in n]
    d2h = [n for n in names if "DtoH" in n]
    assert len(h2d) == 1 and len(d2h) == 1, (h2d, d2h)
    losses = step.losses()
    assert set(losses) == {"total", "spc", "mi", "cmi", "cchunk", "lps", "mfcc", "prosody"}
    assert all(np.isfinite(v) for v in losses.values())


def test_graphed_encoder_step_follows_lr_changes():
    """A FlatAdam lr change between two replays of GraphedEncoderStep reaches the captured
    update (the table keeps its address)."""
    from pase_b200.frontend import WaveFe
    cfg = resolve_cfg("cfg/frontend/PASE+.cfg")
    x = seeded_randn((2, 1, 6400), 5, 0.5)
    cot = seeded_randn((2, 256, 40), 6).cuda()
    loss_fn = lambda y: (y * cot).mean() + y.abs().mean()       # noqa: E731
    lrs = [1e-3, 3e-4, 5e-5, 2e-3]

    def model():
        m = WaveFe(**cfg)
        m.load_state_dict(fill_state_dict(m.state_dict(), 3))
        m = m.cuda().train()
        return m, FlatAdam(m.parameters(), lr=lrs[0])
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    try:
        me, oe = model()
        for k in range(3 + len(lrs)):               # warm-up steps at lrs[0], then one per lr
            oe.param_groups[0]["lr"] = lrs[max(k - 3, 0)]
            oe.zero_grad(set_to_none=True)
            loss_fn(me(x.cuda())).backward()
            oe.step()
        mg, og = model()
        gs = GraphedEncoderStep(mg, og, loss_fn, (2, 1, 6400), "cuda", stream=side, warmup=3,
                                x_init=x)
        for lr in lrs:
            og.param_groups[0]["lr"] = lr
            gs.step()
        torch.cuda.synchronize()
        assert torch.equal(og.flat_param, oe.flat_param)
        assert torch.equal(og.exp_avg_sq, oe.exp_avg_sq)
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())


@pytest.mark.parametrize("ci", range(len(SPC_CASES)))
def test_spc_kernels_equal_the_torch_gather(ci):
    case = SPC_CASES[ci]
    B, T, C, N, sp, _ = case
    frames = _frames(case, ci)
    gen = torch.Generator().manual_seed(ci)
    x = torch.randn(B * T, C, generator=gen)
    g = torch.randn(2 * B, (N + 1) * C, generator=gen)
    ref_y, ref_dx = spc_reference(x.cuda(), g.cuda(), case, frames)
    xr = x.cuda().requires_grad_(True)
    y = Fn.spc_gather(xr, B, T, N, sp, frames)
    y.backward(g.cuda())
    assert torch.equal(y, ref_y) and torch.equal(xr.grad, ref_dx)
    # the device-table form a captured step uses
    t = torch.tensor(frames, dtype=torch.int64, device="cuda")
    assert torch.equal(Fn.spc_gather(x.cuda(), B, T, N, sp, t), ref_y)


def test_spc_kernels_strided_rows():
    check_strided_rows("cuda")


def test_caller_work_after_a_call_sees_the_finished_step(corpus):
    """Eager work queued on the caller's stream right after a call, with no synchronise: an
    eval pass that first runs other shapes until the training shape's encoder plan is evicted
    from the cache, then the training shape itself (whose plan buffers the step used), and a
    copy of the parameters; then one more step.  Everything equals the same sequence run
    eagerly."""
    B, T, steps = 4, 16000, 5
    shapes = [(1, 3200), (2, 3200), (1, 4800), (2, 4800), (1, 6400), (3 * B, T)]
    xs = [seeded_randn((n, 1, t), 20 + i, 0.5).cuda() for i, (n, t) in enumerate(shapes)]
    batches = _batches(len(WavPool(corpus["data_root"], corpus["cfg"], "train", placement="cpu")),
                       B, steps + 1, 13)

    def probe(model, engine):
        snap = engine.flat_param.clone()
        model.eval()
        with torch.no_grad():
            outs = [model.frontend(x).clone() for x in xs]
        model.train()
        return snap, outs

    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        model, engine, batcher = _setup(corpus, "pase", T, "3xf16")
        _seed(8)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                batcher.reset()
            if k == steps:
                ref = probe(model, engine)
            engine.zero_grad(set_to_none=True)
            _, _, preds, labels = model(batcher(idx))
            tot, _ = total_loss(model, preds, labels)
            tot.backward()
            engine.step()
        gmodel, gengine, gbatcher = _setup(corpus, "pase", T, "3xf16")
        step = GraphedTrainStep(gmodel, gengine, gbatcher, B)
        _seed(8)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                gbatcher.reset()
            if k == steps:
                plans = gmodel.frontend._plans
                captured = next(p for key, p in plans.items() if key[:2] == (3 * B, T))
                got = probe(gmodel, gengine)          # right after a replay, no synchronise
                # the eval pass evicted the captured plan and built a new one for its shape;
                # the step still holds the captured one
                now = next(p for key, p in plans.items() if key[:2] == (3 * B, T))
                assert now is not captured and any(p is captured for p in step._plans)
            step(idx)
        torch.cuda.synchronize()
        assert torch.equal(got[0], ref[0])
        for a, b in zip(got[1], ref[1]):
            assert torch.equal(a, b)
        _compare(engine, gengine)
    finally:
        Fn.set_precision(prev)


def test_spc_kernels_refuse_bad_arguments():
    x = torch.zeros(2 * 44, 8, device="cuda")
    fr = torch.tensor([22, 38, 5], dtype=torch.int64, device="cuda")
    out = torch.zeros(4, 48, device="cuda")
    good = [x, 8, fr, 2, 44, 8, 5, 16, out]
    _lib.call("pase_spc_gather", *good)
    for i, v, msg in [(0, None, "x is NULL"), (2, None, "frames is NULL"), (8, None, "out is NULL"),
                      (3, 0, "B="), (5, 0, "C="), (6, -1, "N="), (1, 7, "ldx"),
                      (4, 43, "no current frame")]:
        args = list(good)
        args[i] = v
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("pase_spc_gather", *args)
    g = torch.zeros(4, 48, device="cuda")
    dx = torch.zeros(2 * 44, 8, device="cuda")
    bgood = [g, fr, 2, 44, 8, 5, 16, dx]
    _lib.call("pase_spc_gather_bwd", *bgood)
    for i, v, msg in [(0, None, "g is NULL"), (1, None, "frames is NULL"), (7, None, "dx is NULL"),
                      (2, 70000, "B="), (3, 43, "no current frame")]:
        args = list(bgood)
        args[i] = v
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("pase_spc_gather_bwd", *args)
    torch.cuda.synchronize()
