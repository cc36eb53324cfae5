"""The captured PASE/PASE+ training step (pase_b200/graph.py GraphedTrainStep), CPU side: the
planner draws what the eager loop draws and in its order, every refusal names what it refuses,
the emulated SPC gather kernels equal the torch gather SPCMinion used before them, and the flat
Adam hyper-parameter table keeps its address across lr changes.
"""
import copy
import json
import os
import random

import numpy as np
import pytest
import torch

import emul
from helpers import resolve_cfg
from pase_b200 import functional as Fn
from pase_b200 import ops
from pase_b200.batch import DeviceBatcher, FeaturePool, WavPool
from pase_b200.graph import GraphedTrainStep, TrainPlanner, spc_minions
from pase_b200.minions import SPCMinion
from pase_b200.optim import FlatAdam
from pase_b200.pase import pase
from pase_b200.utils import parse_workers

HOP = 160


def _mlp(name, nout, **kw):
    d = {"num_outputs": nout, "dropout": 0, "hidden_size": 256, "hidden_layers": 1, "name": name,
         "loss": "MSELoss", "skip": False}
    d.update(kw)
    return d


def _decoder():
    return {"num_outputs": 1, "dropout": 0, "dropout_time": 0.0, "hidden_layers": 1,
            "name": "cchunk", "type": "decoder", "hidden_size": 64, "fmaps": [512, 256, 128],
            "strides": [4, 4, 10], "kwidths": [30, 30, 30], "loss": "L1Loss"}


def _cls(name, **kw):
    d = {"num_outputs": 1, "dropout": 0, "hidden_size": 256, "hidden_layers": 1, "name": name,
         "loss": "BCEWithLogitsLoss", "skip": False}
    d.update(kw)
    return d


# cfg/workers/workers.cfg (the PASE recipe, with PASE.cfg) and cfg/workers/workers+.cfg (PASE+),
# transforms included: DeviceBatcher.from_train_opts reads them
WORKERS = {
    "regr": [_decoder(), _mlp("lps", 1025, transform={"der_order": 0}),
             _mlp("mfcc", 20, transform={"der_order": 0, "order": 20}),
             _mlp("prosody", 4, transform={"der_order": 0})],
    "cls": [_cls("spc", type="spc"), _cls("mi"), _cls("cmi")],
}
WORKERS_KEYS = {"mfcc": 20, "prosody": 4}
_R7 = dict(context=1, r=7)
WORKERS_PLUS = {
    "regr": [_decoder(), _mlp("lps", 3075, **_R7),
             _mlp("lps_long", 3075, transform={"win": 512}, **_R7),
             _mlp("fbank", 120, **_R7),
             _mlp("fbank_long", 120, transform={"win": 1024, "n_fft": 1024}, **_R7),
             _mlp("gtn", 120, **_R7), _mlp("gtn_long", 120, transform={"win": 2048}, **_R7),
             _mlp("mfcc", 39, **_R7),
             _mlp("mfcc_long", 60, transform={"win": 2048, "order": 20}, **_R7),
             _mlp("prosody", 12, **_R7)],
    "cls": [_cls("mi"), _cls("cmi", augment=True)],
}
PLUS_KEYS = {"fbank": 120, "fbank_long": 120, "gtn": 120, "gtn_long": 120, "mfcc": 39,
             "mfcc_long": 60, "prosody": 12}
RECIPES = {"pase": ("cfg/frontend/PASE.cfg", WORKERS, WORKERS_KEYS),
           "pase+": ("cfg/frontend/PASE+.cfg", WORKERS_PLUS, PLUS_KEYS)}


def build_corpus(root, n, min_len, max_len, seed=2026):
    """`n` int16 utterances of min_len..max_len samples in LibriSpeech-style prefix groups, with
    cached features for the keys of both recipes (under cache_<recipe>/train/<key>)."""
    from scipy.io import wavfile
    rng = np.random.RandomState(seed)
    data_root = os.path.join(root, "wavs")
    os.makedirs(data_root)
    data = []
    for i in range(n):
        name = "%d-%d-%04d-%d.wav" % (100 + i // 8, 3, i // 4, i % 4)
        L = int(rng.randint(min_len, max_len + 1))
        wavfile.write(os.path.join(data_root, name), 16000, (rng.randn(L) * 3000).astype(np.int16))
        for recipe, (_, _, keys) in RECIPES.items():
            for k, F in keys.items():
                d = os.path.join(root, "cache_" + recipe, "train", k)
                os.makedirs(d, exist_ok=True)
                torch.save(torch.from_numpy(rng.randn(F, L // HOP + 1).astype(np.float32)),
                           os.path.join(d, os.path.splitext(name)[0] + "." + k))
        data.append({"filename": name})
    cfg = os.path.join(root, "cfg.json")
    with open(cfg, "w") as fh:
        json.dump({"train": {"data": data}}, fh)
    return data_root, cfg


def make_model(recipe, seed=0):
    fe, wcfg, _ = RECIPES[recipe]
    torch.manual_seed(seed)
    return pase(frontend_cfg=resolve_cfg(fe), minions_cfg=parse_workers(copy.deepcopy(wcfg)))


# ---------------------------------------------------------------- SPC gather


def _torch_gather(x, B, T, N, t, ft, pt):
    """What SPCMinion.forward computed before the gather kernels (minions.py:609-627)."""
    v = x.view(B, T, -1)
    fut = v[:, ft:ft + N].transpose(1, 2).reshape(B, -1)
    past = v[:, pt - N:pt].transpose(1, 2).reshape(B, -1)
    cur = v[:, t]
    return torch.cat([torch.cat([cur, fut], 1), torch.cat([cur, past], 1)], 0).contiguous()


# (B, T', C, N, seq_pad, frames): the bounds of every range, and seq_pad = 0 with future_t = t
SPC_CASES = [
    (3, 100, 20, 5, 16, None),
    (2, 44, 8, 5, 16, (22, 38, 5)),            # t = M + 1, future_t = t + seq_pad, past_t = N
    (4, 60, 12, 5, 16, (38, 54, 21)),          # t = T - M - 1, future_t = T - N - 1, past_t max
    (2, 30, 4, 3, 0, (10, 10, 9)),             # seq_pad = 0: the fut window starts at t
    (5, 200, 100, 5, 16, None),
    (1, 9, 3, 1, 2, (4, 6, 1)),
]


def _frames(case, seed):
    B, T, C, N, sp, frames = case
    if frames is None:
        m = SPCMinion(C, 1, 0, hidden_size=4, hidden_layers=1, ctxt_frames=N, seq_pad=sp)
        frames = m.draw_frames(T, random.Random(seed))
    return frames


def spc_reference(x, g, case, frames):
    """(forward, backward) of the torch gather for upstream gradient g."""
    B, T, C, N, sp, _ = case
    xr = x.clone().requires_grad_(True)
    y = _torch_gather(xr, B, T, N, *frames)
    y.backward(g)
    return y.detach(), xr.grad


def check_strided_rows(device):
    """Rows with a row stride larger than C and a storage offset (a column slice of a wider
    matrix) against the torch gather, forward and backward."""
    B, T, C, N, sp, frames = 3, 60, 12, 5, 16, (30, 47, 10)
    gen = torch.Generator().manual_seed(7)
    base = torch.randn(B * T, C + 5, generator=gen).to(device)
    g = torch.randn(2 * B, (N + 1) * C, generator=gen).to(device)
    ref = base.clone().requires_grad_(True)
    y_ref = _torch_gather(ref[:, 2:2 + C], B, T, N, *frames)
    y_ref.backward(g)
    got = base.clone().requires_grad_(True)
    y = Fn.spc_gather(got[:, 2:2 + C], B, T, N, sp, frames)
    y.backward(g)
    assert torch.equal(y, y_ref.detach()) and torch.equal(got.grad, ref.grad)


def test_emulated_spc_gather_strided_rows(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    check_strided_rows("cpu")


@pytest.mark.parametrize("ci", range(len(SPC_CASES)))
def test_emulated_spc_gather_matches_torch_gather(ci, monkeypatch):
    case = SPC_CASES[ci]
    B, T, C, N, sp, _ = case
    frames = _frames(case, ci)
    gen = torch.Generator().manual_seed(ci)
    x = torch.randn(B * T, C, generator=gen)
    g = torch.randn(2 * B, (N + 1) * C, generator=gen)
    ref_y, ref_dx = spc_reference(x, g, case, frames)
    monkeypatch.setattr(ops, "call", emul.call)
    xr = x.clone().requires_grad_(True)
    y = Fn.spc_gather(xr, B, T, N, sp, frames)
    y.backward(g)
    assert torch.equal(y, ref_y) and torch.equal(xr.grad, ref_dx)


@pytest.mark.parametrize("bad", [(21, 38, 5), (39, 55, 5), (22, 37, 5), (22, 39, 5), (22, 38, 4),
                                 (22, 38, 6)])
def test_spc_frames_out_of_range_are_refused_before_any_launch(bad, monkeypatch):
    # T' = 44, N = 5, seq_pad = 16: t in [22, 23), future_t in [t + 16, 39), past_t in [5, t - 16)
    calls = []
    monkeypatch.setattr(ops, "call", lambda name, *a: calls.append(name))
    x = torch.zeros(2 * 44, 8)
    with pytest.raises(ValueError, match="outside the ranges"):
        Fn.spc_gather(x, 2, 44, 5, 16, bad)
    assert calls == []


def test_planner_draws_what_eager_spc_forward_consumes(monkeypatch):
    seen = []

    def spy(name, *a):
        if name == "pase_spc_gather":
            seen.append(tuple(a[2].tolist()))
        return emul.call(name, *a)
    monkeypatch.setattr(ops, "call", spy)
    from pase_b200.minions import cls_worker_maker
    from pase_b200.losses import ContextualizedLoss
    w = cls_worker_maker({"num_outputs": 1, "dropout": 0, "hidden_size": 8, "hidden_layers": 1,
                          "name": "spc", "type": "spc", "skip": False,
                          "loss": ContextualizedLoss("BCEWithLogitsLoss")}, 12)
    m = w.minion
    x = torch.randn(3, 12, 100)
    random.seed(9)
    for _ in range(4):
        w(x, 1)
    rng = random.Random(9)
    assert seen == [m.draw_frames(100, rng) for _ in range(4)]


# ---------------------------------------------------------------- planner and refusals


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("train_corpus"))
    return build_corpus(root, 24, 9000, 20000)


def _cpu_batcher(corpus, recipe, T):
    data_root, cfg = corpus
    wavs = WavPool(data_root, cfg, "train", placement="cpu")
    cache = os.path.join(os.path.dirname(data_root), "cache_" + recipe)
    wcfg = RECIPES[recipe][1]
    cached = {k: (FeaturePool(cache, "train", k, wavs.names, "cpu"), HOP)
              for k in RECIPES[recipe][2]}
    return DeviceBatcher(wavs, T, mi=True, random_scale=True, cached=cached,
                         order=[w["name"] for ws in wcfg.values() for w in ws
                                if w["name"] in cached])


def _eager_draws(model, batcher, batches, T):
    """The eager loop's host draws with the global generators: batcher(indices) draws the
    plan (its kernels are emulated), then model(batch) draws the SPC frames; the SPC heads run
    on random rows here, the rest of the model does not draw."""
    spc = spc_minions(model)
    gen = torch.Generator().manual_seed(0)
    out = []
    for idx in batches:
        plan = batcher.plan(idx)
        batcher.run(torch.from_numpy(plan.table))
        frames = []
        for m in spc:
            n0 = len(_SEEN)
            m(torch.randn(len(idx), model.frontend.emb_dim, T, generator=gen), 1)
            frames += list(_SEEN[n0])
        out.append(np.concatenate([plan.table, np.asarray(frames, np.int64)]))
    return out


_SEEN = []


@pytest.fixture()
def emulated(monkeypatch):
    def call(name, *a):
        if name == "pase_spc_gather":
            _SEEN.append(tuple(a[2].tolist()))
        return emul.call(name, *a)
    monkeypatch.setattr(ops, "call", call)
    yield


BATCHES = [[3, 7, 1, 12], [20, 5, 9, 14], [0, 22, 17, 8]]


def test_draw_order_across_steps_matches_the_eager_loop(corpus, emulated):
    model = make_model("pase")
    T = 8000
    batcher = _cpu_batcher(corpus, "pase", T)
    assert len(spc_minions(model)) == 1
    random.seed(4)
    np.random.seed(4)
    torch.manual_seed(4)
    eager = _eager_draws(model, batcher, BATCHES, 50)
    planner = TrainPlanner(model, batcher)
    assert planner.Tq == 50
    for rng in (None, "triple"):
        batcher.reset()
        if rng is None:
            random.seed(4)
            np.random.seed(4)
            torch.manual_seed(4)
        else:
            rng = (random.Random(4), np.random.RandomState(4), torch.Generator().manual_seed(4))
        for idx, ref in zip(BATCHES, eager):
            _, table = planner(idx, rng)
            assert np.array_equal(table, ref)


def test_refusals(corpus):
    import torch.distributed as dist
    model = make_model("pase")
    batcher = _cpu_batcher(corpus, "pase", 8000)

    def engine(**kw):
        return FlatAdam(list(model.parameters()), lr=1e-3, **kw)
    eng = engine().bind_encoder(model.frontend)
    with pytest.raises(ValueError, match="eval mode"):
        GraphedTrainStep(model.eval(), eng, batcher, 4)
    model.train()
    with pytest.raises(TypeError, match="FlatAdam"):
        GraphedTrainStep(model, torch.optim.Adam(model.parameters()), batcher, 4)
    with pytest.raises(ValueError, match="bind_encoder"):
        GraphedTrainStep(model, engine(), batcher, 4)
    with pytest.raises(ValueError, match="warmup"):
        GraphedTrainStep(model, eng, batcher, 4, warmup=0)
    with pytest.raises(ValueError, match="batch_size"):
        GraphedTrainStep(model, eng, batcher, 0)
    # 4000 samples -> T' = 25 frames: SPC's range(22, 4) for the current frame is empty
    with pytest.raises(ValueError, match="no current frame"):
        GraphedTrainStep(model, eng, _cpu_batcher(corpus, "pase", 4000), 4)
    with pytest.raises(ValueError, match="CUDA"):
        GraphedTrainStep(model, eng, batcher, 4)
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        peer = engine(peer_dp=True).bind_encoder(model.frontend)
    finally:
        dist.destroy_process_group()
    with pytest.raises(NotImplementedError, match="peer_dp"):
        GraphedTrainStep(model, peer, batcher, 4)


def test_spc_head_refuses_a_chunk_too_short_for_its_frames():
    m = SPCMinion(8, 1, 0, hidden_size=4, hidden_layers=1)
    assert not m.frames_ok(43) and m.frames_ok(44)
    with pytest.raises(ValueError, match="empty"):
        m.draw_frames(43)


# ---------------------------------------------------------------- flat Adam table


def test_flat_adam_table_keeps_its_address(monkeypatch):
    import emul
    monkeypatch.setattr(ops, "call", emul.call)
    net = torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.Linear(7, 3))
    opt = FlatAdam([{"params": list(net[0].parameters()), "lr": 1e-2},
                    {"params": list(net[1].parameters())}], lr=1e-3)
    t0 = opt._segments()
    ptr, before = t0.data_ptr(), t0.clone()
    for k, lr in enumerate((5e-3, 2e-3, 1e-4)):
        opt.param_groups[k % 2]["lr"] = lr
        opt.param_groups[1]["betas"] = (0.8, 0.99)
        net(torch.randn(4, 5)).square().mean().backward()
        opt.step()
        t = opt._segments()
        assert t.data_ptr() == ptr
        lrs = t.view(torch.float32).view(-1, 12)[:, 4]         # rows {a, b, lr, beta1, ...}
        assert lrs.tolist() == [np.float32(g["lr"]) for g in opt.param_groups]
    assert not torch.equal(t, before)
