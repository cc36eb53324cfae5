"""AMI close-talk/distant-mic batch assembly (DeviceBatcher with dataset='ami') on the GPU:
the reference's collated batches bit for bit with the corpus in HBM and in mapped page-locked
host memory, graph replay with new plans, launch counts that do not depend on the draws (the
alias and padded windows included), and GraphedTrainStep / GraphedEvalStep on a paired pool
equal to the eager loop and pass.
"""
import json
import os
import random

import numpy as np
import pytest
import torch

from ami_corpus import CASES, HOP, SPLIT
from batch_corpus import digest
from distortion_banks import build_banks, case_cfg
from helpers import GOLDEN, fill_state_dict
from pase_b200 import ops
from pase_b200 import functional as Fn
from pase_b200.batch import DeviceBatcher, WavPool
from pase_b200.distortions import config_distortions
from pase_b200.graph import GraphedEvalStep, GraphedTrainStep
from pase_b200.optim import FlatAdam
from pase_b200.pase import total_loss
from pase_b200.targets import LPS
from test_ami_batch import ami_batcher
from test_batch import _check_batch, _seed
from test_eval_step_gpu import _assert_equal, _eager_pass, _graphed_pass
from test_train_step import RECIPES, make_model
from test_train_step_gpu import _batches, _compare, _poly

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    from ami_corpus import build_ami_corpus
    root = str(tmp_path_factory.mktemp("ami_corpus_gpu"))
    data_root, cfg, cache = build_ami_corpus(root)
    banks = build_banks(os.path.join(root, "banks"))
    return dict(root=root, data_root=data_root, cfg=cfg, cache=cache, banks=banks)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ami_batch.pt"))


@pytest.mark.parametrize("placement", ["cuda", "pinned"])
@pytest.mark.parametrize("case", list(CASES))
def test_golden_hashes(case, placement, corpus, golden):
    meta = json.loads(golden[case + "/meta"])
    b = ami_batcher(corpus, case, device="cuda", placement=placement)
    _seed(CASES[case]["seed"])
    for bi, idx in enumerate(CASES[case]["batches"]):
        out = b(idx)
        torch.cuda.synchronize()
        _check_batch(out, meta["arrays"][bi], case, golden.get("%s/%d/chunk" % (case, bi)))


def _full_batcher(corpus):
    return ami_batcher(corpus, "pair_mi_dist", device="cuda", placement="cuda",
                       targets=[LPS(hop=HOP, name="lps"), LPS(hop=HOP, win=512, name="lps_long")])


def _plan(b, ix, seed):
    b.reset()
    g = torch.Generator()
    g.manual_seed(seed)
    return b.plan(ix, rng=(random.Random(seed), np.random.RandomState(seed), g))


def test_graph_replay_with_new_plans(corpus):
    b = _full_batcher(corpus)
    plans = [_plan(b, ix, 40 + i) for i, ix in enumerate([[2, 6, 10, 4], [5, 8, 0, 9],
                                                           [1, 3, 7, 10]])]
    table = b.upload(plans[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                   # warm-up outside the capture
        b.run(table)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = b.run(table)
    for p in plans[1:]:
        b.upload(p, out=table)
        graph.replay()
        torch.cuda.synchronize()
        ref = b.run(b.upload(p))
        torch.cuda.synchronize()
        assert set(out) == set(ref)
        for k in ref:
            assert digest(out[k].cpu().numpy()) == digest(ref[k].cpu().numpy()), k


def test_launch_count_does_not_depend_on_the_draws(corpus):
    b = _full_batcher(corpus)
    b([2, 6])                                    # the first call builds the LPS constants
    counts, kinds = [], set()
    for seed in range(1, 7):
        plan = _plan(b, [2, 6, 10, 4, 1], seed)
        if seed == 6:                            # no distortion drawn at all
            plan = b._pack([dict(s, distortions={}) for s in plan.samples])
        kinds |= {"alias" if s["paired"] is None else s["paired"][1] for s in plan.samples}
        t = b.upload(plan)
        n0 = ops.launch_count
        b.run(t)
        counts.append(ops.launch_count - n0)
    torch.cuda.synchronize()
    assert len(set(counts)) == 1, counts
    assert "alias" in kinds and len(kinds) >= 2, kinds


# ---------------------------------------------------------------- graphed steps on a paired pool


def _paired_train_corpus(root, split, n, seed):
    """`n` int16 close-talk utterances of 32001..64000 samples with distant-mic channels '1'
    and '2' (some shorter than the chunk's end, some far shorter), and cached features of the
    close-talk utterances for the keys of both recipes (under cache_<recipe>/<split>/<key>)."""
    from scipy.io import wavfile
    rng = np.random.RandomState(seed)
    data_root = os.path.join(root, "wavs")
    for d in ("ihm", "sdm1", "sdm2"):
        os.makedirs(os.path.join(data_root, d), exist_ok=True)
    data = []
    for i in range(n):
        name = "%d-%d-%04d-%d.wav" % (100 + i // 8, 3, i // 4, i % 4)
        L = int(rng.randint(32001, 64001))
        wavfile.write(os.path.join(data_root, "ihm", name), 16000,
                      (rng.randn(L) * 3000).astype(np.int16))
        entry = {"filename": "ihm/" + name}
        for c in ("1", "2"):
            M = L - int(rng.choice([0, 40, 9000, L - 20000]))
            wavfile.write(os.path.join(data_root, "sdm" + c, name), 16000,
                          (rng.randn(M) * 2000).astype(np.int16))
            entry[c] = "sdm%s/%s" % (c, name)
        data.append(entry)
        for recipe, (_, _, keys) in RECIPES.items():
            for k, F in keys.items():
                d = os.path.join(root, "cache_" + recipe, split, k)
                os.makedirs(d, exist_ok=True)
                torch.save(torch.from_numpy(rng.randn(F, L // HOP + 1).astype(np.float32)),
                           os.path.join(d, os.path.splitext(name)[0] + "." + k))
    cfg = os.path.join(root, "cfg.json")
    with open(cfg, "w") as fh:
        json.dump({split: {"data": data}}, fh)
    return data_root, cfg


@pytest.fixture(scope="module")
def paired(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("ami_train_gpu"))
    data_root, cfg = _paired_train_corpus(root, "train", 24, 77)
    return dict(root=root, data_root=data_root, cfg=cfg,
                banks=build_banks(os.path.join(root, "banks")))


def _setup(paired, recipe, T, seed=5):
    fe, wcfg, _ = RECIPES[recipe]
    model = make_model(recipe)
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    model.frontend.precision = "3xf16"
    model = model.cuda().train()
    groups = [{"params": list(model.frontend.parameters())}]
    groups += [{"params": list(w.parameters())} for w in
               list(model.classification_workers) + list(model.regression_workers)]
    engine = FlatAdam(groups, lr=5e-4).bind_encoder(model.frontend)
    wavs = WavPool(paired["data_root"], paired["cfg"], "train", placement="cuda", ihm2sdm="1,2")
    dist = None
    if recipe == "pase+":
        dist = config_distortions(device="cuda", **case_cfg("pase_plus", paired["banks"])[0])
    batcher = DeviceBatcher.from_train_opts(
        wcfg, T, HOP, wavs, random_scale=True, distortions=dist,
        trans_cache=os.path.join(paired["root"], "cache_" + recipe),
        dataset="AmiSegTupleWavDataset", ihm2sdm="1,2")
    return model, engine, batcher


@pytest.mark.parametrize("recipe", ["pase+", "pase"])
def test_graphed_steps_equal_the_eager_loop(recipe, paired):
    B, T, steps = 4, 16000, 6
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        batches = _batches(24, B, steps, 11)
        model, engine, batcher = _setup(paired, recipe, T)
        _seed(3)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                batcher.reset()
            _poly(engine, k, steps)
            engine.zero_grad(set_to_none=True)
            _, _, preds, labels = model(batcher(idx))
            tot, losses = total_loss(model, preds, labels)
            tot.backward()
            engine.step()
        eager = dict({n: float(v.detach()) for n, v in losses.items()}, total=float(tot.detach()))
        torch.cuda.synchronize()
        gmodel, gengine, gbatcher = _setup(paired, recipe, T)
        step = GraphedTrainStep(gmodel, gengine, gbatcher, B)
        _seed(3)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                gbatcher.reset()
            _poly(gengine, k, steps)
            step(idx)
        assert step.graph is not None and step.calls == steps
        got = step.losses()
        torch.cuda.synchronize()
        assert set(got) == set(eager)
        for n in eager:
            assert got[n] == eager[n], (n, got[n], eager[n])
        _compare(engine, gengine)
    finally:
        Fn.set_precision(prev)


def test_graphed_eval_pass_equals_the_eager_pass(paired):
    B, T, nb = 4, 16000, 5
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        batches = _batches(24, B, nb, 17)
        model, _, batcher = _setup(paired, "pase+", T)
        model.eval()
        _seed(4)
        eager = _eager_pass(model, batcher, batches, None)
        gmodel, _, gbatcher = _setup(paired, "pase+", T)
        gmodel.eval()
        ev = GraphedEvalStep(gmodel, gbatcher, B, max_batches=nb)
        _seed(4)
        got = _graphed_pass(ev, gbatcher, batches, None)
        assert ev.graph is not None and ev.calls == nb
        _assert_equal(got, eager)
    finally:
        Fn.set_precision(prev)
