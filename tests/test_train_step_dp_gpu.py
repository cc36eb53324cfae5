"""The data-parallel captured training step and validation pass on the GPU, against W replicas
in one process on one GPU.

Each rank of a spawned process group builds its own replica (aligned to rank 0's weights),
engine, batchers and generator triple, and runs GraphedTrainStep(group=...) on its shard of
the indices (DistributedSampler, shared seed and epoch): 1 eager warm-up step and 3 replays.
The reference runs every rank's eager step on one replica each, with a plain
FlatAdam(grad_scale=1/W), and puts the rank-ordered fp32 sum of the replicas' flat gradients
into every replica before its update: the arithmetic of pase_adam_flat_dp (a rank-ordered sum,
then x 1/W) and, for W = 2, of the gloo fallback (sum, x 1/2, exact).  Expected bit for bit:
the parameters on every rank, each rank's BatchNorm running statistics, ``losses()`` (the mean
of the replicas' losses); the DP validation pass against an eager pass of rank 0's model over
every rank's batches; rank 0's consolidated Adam state, and the step a run resumed from the
Saver files takes.

Two GPUs with the peer engine (NCCL process group, one replay per step; skipped below two
GPUs), and two processes on one GPU with a plain engine over gloo (two replays per step, the
all-reduce between them).
"""
import os
import random
import socket

import numpy as np
import pytest
import torch

from distortion_banks import build_banks, case_cfg
from helpers import fill_state_dict
from test_train_step import RECIPES, build_corpus, make_model

pytestmark = pytest.mark.gpu

HOP = 160
B, T, W = 4, 16000, 2
STEPS = 4                 # 1 eager warm-up + capture + 2 more replays; the 5th is the resumed one
EVAL_BATCHES = 3
LR = 5e-4


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("train_step_dp_gpu"))
    data_root, cfg = build_corpus(root, 40, 32001, 64000)
    return dict(root=root, data_root=data_root, cfg=cfg,
                banks=build_banks(os.path.join(root, "banks")))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _triple(s):
    return (random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def _modules(model):
    """(name, module) per FlatAdam group: the frontend, then every worker."""
    return [("frontend", model.frontend)] + [
        (w.name, w) for w in list(model.classification_workers) + list(model.regression_workers)]


def _model(recipe, precision, seed):
    model = make_model(recipe)
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    model.frontend.precision = precision
    return model.cuda().train()


def _engine(model, **kw):
    from pase_b200.optim import FlatAdam
    groups = [{"params": list(m.parameters())} for _, m in _modules(model)]
    return FlatAdam(groups, lr=LR, **kw).bind_encoder(model.frontend)


def _batcher(corpus, recipe):
    from pase_b200.batch import DeviceBatcher, WavPool
    from pase_b200.distortions import config_distortions
    wavs = WavPool(corpus["data_root"], corpus["cfg"], "train", placement="cuda")
    dist = None
    if recipe == "pase+":
        dist = config_distortions(device="cuda", **case_cfg("pase_plus", corpus["banks"])[0])
    return DeviceBatcher.from_train_opts(
        RECIPES[recipe][1], T, HOP, wavs, random_scale=True, distortions=dist,
        trans_cache=os.path.join(corpus["root"], "cache_" + recipe))


def _shard(n, rank, seed):
    """Rank `rank`'s batches of epoch 0: DistributedSampler(shuffle, drop_last), then B."""
    from torch.utils.data import BatchSampler, DistributedSampler
    s = DistributedSampler(range(n), num_replicas=W, rank=rank, shuffle=True, seed=seed,
                           drop_last=True)
    s.set_epoch(0)
    return [list(b) for b in BatchSampler(s, B, drop_last=True)]


def _bn(model):
    return {k: v.clone().cpu() for k, v in model.state_dict().items() if "running" in k}


def _rank(rank, backend, port, recipe, precision, corpus, out):
    import torch.distributed as dist
    from pase_b200 import functional as Fn
    from pase_b200.dp import broadcast_parameters_and_buffers
    from pase_b200.graph import GraphedEvalStep, GraphedTrainStep
    from pase_b200.modules import Saver
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    peer = backend == "nccl"
    dev = torch.device("cuda", rank if peer else 0)
    torch.cuda.set_device(dev)
    if peer:
        dist.init_process_group("nccl", rank=rank, world_size=W, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=W)
    group = dist.group.WORLD
    Fn.set_precision(precision)
    try:
        n = len(corpus_names(corpus))
        model = _model(recipe, precision, 5 + rank)         # replicas start different ...
        broadcast_parameters_and_buffers(model)             # ... and are aligned to rank 0
        engine = _engine(model, peer_dp=True) if peer else _engine(model)
        assert (engine._peer is not None) == peer
        batcher = _batcher(corpus, recipe)
        batches = _shard(n, rank, 11)
        rng = _triple(100 + rank)
        step = GraphedTrainStep(model, engine, batcher, B, warmup=1, group=group)
        assert step.split == (not peer)
        batcher.reset()
        losses = []
        for idx in batches[:STEPS]:
            step(idx, rng)
            losses.append(step.losses())
        assert step.graph is not None and step.calls == STEPS
        assert (step.graph_b is not None) == (not peer)
        torch.cuda.synchronize()
        res = dict(flat=engine.flat_param.cpu(), bn=_bn(model), losses=losses)

        # validation: every rank its own batches, rank 0's running statistics
        model.eval()
        ev = GraphedEvalStep(model, _batcher(corpus, recipe), B, max_batches=EVAL_BATCHES,
                             warmup=1, group=group)
        vrng = _triple(200 + rank)
        for idx in _shard(n, rank, 12)[:EVAL_BATCHES]:
            ev(idx, vrng)
        res["eval"] = ev.losses()
        res["bn_after_eval"] = _bn(model)
        if not peer:
            # a rank that ran another number of batches fails the gather on every rank
            ev.reset()
            ev.batcher.reset()
            for idx in _shard(n, rank, 12)[:1 + rank]:
                ev(idx, vrng)
            with pytest.raises(RuntimeError, match="same number"):
                ev.losses()
        model.train()

        # checkpoint: consolidate on every rank, rank 0 saves, every rank resumes
        engine.consolidate_state()
        ck = os.path.join(out, "ckpt")
        if rank == 0:
            res["state"] = engine.state_dict()
            for (name, m), view in zip(_modules(model), engine.views()):
                Saver(m, ck, optimizer=view, prefix=name + "-").save(name, STEPS)
        dist.barrier()
        model2 = _model(recipe, precision, 50 + rank)
        engine2 = _engine(model2, peer_dp=True) if peer else _engine(model2)
        for (name, m), view in zip(_modules(model2), engine2.views()):
            assert Saver(m, ck, optimizer=view, prefix=name + "-").load_weights()
        assert torch.equal(engine2.flat_param, engine.flat_param)
        step2 = GraphedTrainStep(model2, engine2, batcher, B, warmup=1, group=group)
        step2(batches[STEPS], rng)
        res["resumed_loss"] = step2.losses()
        torch.cuda.synchronize()
        res["resumed_flat"] = engine2.flat_param.cpu()
        torch.save(res, os.path.join(out, "rank%d.pt" % rank))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def corpus_names(corpus):
    from pase_b200.batch import WavPool
    return WavPool(corpus["data_root"], corpus["cfg"], "train", placement="cpu").names


def _eager_forward(model, batcher, idx, rng):
    """batcher(idx, rng) and the forward, the SPC heads drawing from rng[0] (the eager heads
    draw from `random`)."""
    batch = batcher(idx, rng)
    saved = random.getstate()
    random.setstate(rng[0].getstate())
    try:
        return model(batch)
    finally:
        rng[0].setstate(random.getstate())
        random.setstate(saved)


def _reference(recipe, precision, corpus):
    """W replicas on one GPU, every update on the rank-ordered sum of their flat gradients."""
    from pase_b200.pase import eval_losses, total_loss
    n = len(corpus_names(corpus))
    reps = []
    for r in range(W):
        model = _model(recipe, precision, 5)
        reps.append(dict(model=model, engine=_engine(model, grad_scale=1.0 / W),
                         batcher=_batcher(corpus, recipe), batches=_shard(n, r, 11),
                         rng=_triple(100 + r)))
        reps[-1]["batcher"].reset()

    def one_step(k):
        dicts = []
        for rep in reps:
            model, engine = rep["model"], rep["engine"]
            engine.zero_grad(set_to_none=True)
            _, _, preds, labels = _eager_forward(model, rep["batcher"], rep["batches"][k],
                                                 rep["rng"])
            tot, losses = total_loss(model, preds, labels)
            tot.backward()
            engine.pack_grads()
            dicts.append(dict({m: float(v.detach()) for m, v in losses.items()},
                              total=float(tot.detach())))
        g = reps[0]["engine"].flat_grad.clone()
        for rep in reps[1:]:
            g += rep["engine"].flat_grad
        for rep in reps:
            rep["engine"].flat_grad.copy_(g)
            rep["engine"].step()
        return {m: sum(d[m] for d in dicts) / W for m in dicts[0]}

    ref = dict(losses=[one_step(k) for k in range(STEPS)])
    torch.cuda.synchronize()
    ref["flat"] = [rep["engine"].flat_param.cpu() for rep in reps]
    ref["bn"] = [_bn(rep["model"]) for rep in reps]
    ref["state"] = reps[0]["engine"].state_dict()
    # the eager validation pass of rank 0's model over every rank's batches, rank-major
    model = reps[0]["model"].eval()
    rows = []
    for r in range(W):
        vb, vrng = _batcher(corpus, recipe), _triple(200 + r)
        for idx in _shard(n, r, 12)[:EVAL_BATCHES]:
            with torch.no_grad():
                _, _, preds, labels = _eager_forward(model, vb, idx, vrng)
                tot, losses = eval_losses(model, preds, labels)
            rows.append(dict({m: float(v.reshape(())) for m, v in losses.items()},
                             total=float(tot)))
    ref["eval"] = {m: [row[m] for row in rows] for m in rows[0]}
    ref["eval_bn"] = _bn(model)
    model.train()
    ref["resumed_loss"] = one_step(STEPS)
    torch.cuda.synchronize()
    ref["resumed_flat"] = reps[0]["engine"].flat_param.cpu()
    return ref


def _check(ref, got):
    for r, res in enumerate(got):
        assert torch.equal(res["flat"], ref["flat"][r]), "parameters, rank %d" % r
        assert torch.equal(res["flat"], got[0]["flat"])
        for k, v in ref["bn"][r].items():
            assert torch.equal(res["bn"][k], v), ("running statistics", r, k)
        for k, (a, e) in enumerate(zip(res["losses"], ref["losses"])):
            assert a == e, ("losses() of step %d on rank %d" % (k, r), a, e)
        # the pass evaluates rank 0's statistics, broadcast into every rank's buffers
        for k, v in ref["eval_bn"].items():
            assert torch.equal(res["bn_after_eval"][k], v), ("broadcast statistics", r, k)
        assert list(res["eval"]) == list(ref["eval"])
        for m in ref["eval"]:
            assert res["eval"][m] == ref["eval"][m], ("validation", r, m)
        assert torch.equal(res["resumed_flat"], ref["resumed_flat"]), "resumed step, rank %d" % r
        assert res["resumed_loss"] == ref["resumed_loss"]
    assert any(not torch.equal(ref["bn"][0][k], ref["bn"][1][k]) for k in ref["bn"][0]), \
        "the ranks' running statistics should differ"
    st, es = got[0]["state"], ref["state"]
    assert st["param_groups"] == es["param_groups"]
    assert set(st["state"]) == set(es["state"])
    for i, e in es["state"].items():
        for key in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(st["state"][i][key], e[key]), (i, key)


def _run(backend, recipe, precision, corpus, tmp_path):
    import torch.multiprocessing as mp
    from pase_b200 import functional as Fn
    mp.spawn(_rank, args=(backend, _free_port(), recipe, precision, corpus, str(tmp_path)),
             nprocs=W, join=True)
    got = [torch.load(tmp_path / ("rank%d.pt" % r), weights_only=False) for r in range(W)]
    prev = Fn.PRECISION
    Fn.set_precision(precision)
    try:
        ref = _reference(recipe, precision, corpus)
    finally:
        Fn.set_precision(prev)
    _check(ref, got)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("recipe,precision", [("pase", "3xf16"), ("pase", "bf16"),
                                              ("pase+", "3xf16"), ("pase+", "bf16")])
def test_peer_engine_two_gpus(recipe, precision, corpus, tmp_path):
    _run("nccl", recipe, precision, corpus, tmp_path)


@pytest.mark.parametrize("recipe,precision", [("pase", "3xf16"), ("pase+", "bf16")])
def test_allreduce_fallback_one_gpu(recipe, precision, corpus, tmp_path):
    _run("gloo", recipe, precision, corpus, tmp_path)
