"""RAdam segments of pase_adam_flat / pase_adam_flat_dp on the GPU: the golden trajectories,
state dicts and Saver files of the reference RAdam (tests/test_flat_radam.py's checks on the
kernel); the workers+ layout against a float64 restatement; Adam segments of a mixed table
bit-equal to an all-Adam table; the data-parallel kernel at world = 1 bit-equal to the
single-GPU one; GraphedTrainStep with RAdam groups bit-equal to the eager loop across rho = 5;
and peer_dp with RAdam on two GPUs.
"""
import os
import struct

import numpy as np
import pytest
import torch

import emul
from test_flat_radam import run_golden, saver_interchange, state_roundtrip
from pase_b200 import ops
from pase_b200.optim import FlatAdam

pytestmark = pytest.mark.gpu

# parameters per group of the PASE+ frontend and its workers+ heads (frontend first, then the
# classification and regression workers: 29.7 M in 13 groups)
WORKERS_PLUS = [7832896, 131841, 131841, 8857537, 5597973, 5597973, 281928, 281928, 281928,
                281928, 136209, 173988, 87636]
HYPER = [(5e-4, 0.9, 0.999, 1e-8, 0.0), (4e-4, 0.9, 0.999, 1e-8, 1e-2),
         (1e-3, 0.8, 0.99, 1e-6, 0.0), (2e-4, 0.85, 0.995, 1e-8, 1e-2)]
SENTINEL = 7.25


def _f32(x):
    return float(np.float32(x))


def layout(algos):
    """Segments of the workers+ sizes with ragged ends: each starts at the first multiple of 4
    after the previous one's end, so up to 3 padding elements share its last float4.  An
    odd-sized head goes last, so the buffer ends inside a float4 (the kernel's scalar tail)."""
    rows, off = [], 0
    for k, size in enumerate([WORKERS_PLUS[0]] + WORKERS_PLUS[2:] + [WORKERS_PLUS[1]]):
        a = (off + 3) // 4 * 4
        lr, b1, b2, eps, wd = HYPER[k % len(HYPER)]
        rows.append(dict(start=a, end=a + size, lr=_f32(lr), b1=_f32(b1), b2=_f32(b2),
                         eps=_f32(eps), wd=_f32(wd), algo=float(algos[k]), si=k))
        off = a + size
    return rows, rows[-1]["end"]


def table(rows, device="cuda"):
    raw = b"".join(struct.pack(emul.optim.ROW, r["start"], r["end"], r["lr"], r["b1"], r["b2"],
                               r["eps"], r["wd"], r["algo"], r["si"]) for r in rows)
    return torch.frombuffer(bytearray(raw), dtype=torch.int64).to(device)


def buffers(n, seed, n_alloc=None):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    n_alloc = n if n_alloc is None else n_alloc
    p = torch.randn(n_alloc, device="cuda", generator=gen)
    g = torch.randn(n_alloc, device="cuda", generator=gen) * 1e-2
    m = torch.randn(n_alloc, device="cuda", generator=gen) * 1e-3
    v = torch.rand(n_alloc, device="cuda", generator=gen) * 1e-4
    return p, g, m, v


def restate(rows, p, g, m, v, steps, grad_scale=1.0):
    """float64 restatement of one update: torch.optim.Adam for algorithm 0, the reference
    RAdam (radam.py:21-76) for 1, from the table's fp32 hyper-parameters."""
    p, g, m, v = (x.double().clone() for x in (p, g, m, v))
    for r in rows:
        a, b, t = r["start"], r["end"], float(steps[r["si"]])
        b1, b2, eps, wd, lr = r["b1"], r["b2"], r["eps"], r["wd"], r["lr"]
        gg = g[a:b] * grad_scale
        if r["algo"] == 0.0:
            gg = gg + wd * p[a:b]
        m[a:b] = b1 * m[a:b] + (1 - b1) * gg
        v[a:b] = b2 * v[a:b] + (1 - b2) * gg * gg
        if r["algo"] == 0.0:
            denom = v[a:b].sqrt() / (1 - b2 ** t) ** 0.5 + eps
            p[a:b] -= lr / (1 - b1 ** t) * m[a:b] / denom
            continue
        rect, step, decay = emul.optim.radam_constants(lr, b1, b2, wd, t)
        p[a:b] += decay * p[a:b]
        p[a:b] -= step * (m[a:b] / (v[a:b].sqrt() + eps) if rect else m[a:b])
    return p, m, v


def test_kernel_matches_reference_goldens():
    run_golden("cuda")


def test_kernel_state_dict_both_ways():
    state_roundtrip("cuda")


def test_kernel_facades_and_saver(tmp_path):
    saver_interchange("cuda", tmp_path)


@pytest.mark.parametrize("algos", ["radam", "mixed"])
def test_workers_plus_layout_against_float64(algos):
    """Two updates of the 13-segment workers+ layout with ragged segment ends and a scalar
    tail; the step counts differ per segment so both RAdam branches run, and every segment
    crosses rho = 5 between the launches of some case."""
    codes = [1] * 13 if algos == "radam" else [k % 2 for k in range(13)]
    rows, n = layout(codes)
    assert n % 4 != 0
    tab = table(rows)
    live = torch.zeros(n, dtype=torch.bool, device="cuda")
    for r in rows:
        live[r["start"]:r["end"]] = True
    p, g, m, v = buffers(n, 11)
    for x in (p, m, v):
        x[~live] = SENTINEL
    steps = torch.tensor([float(1 + (k * 5) % 11) for k in range(13)], device="cuda")
    for launch in range(2):
        steps += 1.0
        want = restate(rows, p, g, m, v, steps.cpu())
        p_old, m_old = p.double(), m.double()
        ops.call("pase_adam_flat", p, g, m, v, n, tab, 13, steps, 1.0)
        torch.cuda.synchronize()
        # fp32: a few ulp of the terms of each value, and of the step for p
        bounds = {"p": 3e-7 * p_old.abs() + 1e-5 * (want[0] - p_old).abs(),
                  "m": 3e-7 * (m_old.abs() + g.double().abs() + p_old.abs() * 1e-2),
                  "v": 3e-7 * want[2].abs()}
        for name, got, w in (("p", p, want[0]), ("m", m, want[1]), ("v", v, want[2])):
            assert bool((got[~live] == SENTINEL).all()), (launch, name, "gap written")
            err = (got.double() - w).abs()[live]
            bad = err > bounds[name][live] + 1e-30
            assert not bool(bad.any()), (launch, name, int(bad.sum()), float(err.max()))
        g = torch.randn(n, device="cuda", generator=torch.Generator(device="cuda")
                        .manual_seed(20 + launch)) * 1e-2


def test_mixed_table_adam_segments_bit_equal_to_all_adam():
    mixed = [k % 2 for k in range(13)]
    rows_m, n = layout(mixed)
    rows_a, _ = layout([0] * 13)
    steps = torch.tensor([float(1 + k) for k in range(13)], device="cuda")
    outs = []
    for rows in (rows_m, rows_a):
        p, g, m, v = buffers(n, 5)
        for _ in range(3):
            ops.call("pase_adam_flat", p, g, m, v, n, table(rows), 13, steps, 0.5)
        outs.append((p, m, v))
    for r in rows_m:
        if r["algo"] == 0.0:
            for a, b in zip(*outs):
                assert torch.equal(a[r["start"]:r["end"]], b[r["start"]:r["end"]]), r["si"]
    # and the RAdam segments did something else
    r = rows_m[1]
    assert not torch.equal(outs[0][0][r["start"]:r["end"]], outs[1][0][r["start"]:r["end"]])


def test_dp_kernel_world_one_bit_equal():
    """pase_adam_flat_dp at world = 1 (this rank's own buffers as one-entry peer tables) runs
    the same per-element update as pase_adam_flat: bit-equal for the mixed table."""
    rows, n = layout([k % 2 for k in range(13)])
    n4 = (n + 3) // 4 * 4
    tab = table(rows)
    steps = torch.tensor([float(1 + (k * 5) % 11) for k in range(13)], device="cuda")
    a = buffers(n4, 9)
    b = tuple(x.clone() for x in a)
    flags = torch.zeros(2, dtype=torch.int32, device="cuda")
    sync = torch.zeros(2, dtype=torch.int32, device="cuda")
    peers = lambda t: torch.tensor([t.data_ptr()], dtype=torch.int64, device="cuda")
    for _ in range(3):
        steps += 1.0
        ops.call("pase_adam_flat", a[0], a[1], a[2], a[3], n4, tab, 13, steps, 1.0)
        ops.call("pase_adam_flat_dp", peers(b[0]), peers(b[1]), peers(flags), b[2], b[3], n4,
                 tab, 13, steps, 1, 0, sync[0:1], sync[1:2])
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert int(sync[0]) == 3 and int(sync[1]) == 0


# ---------------------------------------------------------------- the captured training step

@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    from distortion_banks import build_banks
    from test_train_step import build_corpus
    root = str(tmp_path_factory.mktemp("radam_step_gpu"))
    data_root, cfg = build_corpus(root, 40, 32001, 64000)
    return dict(root=root, data_root=data_root, cfg=cfg,
                banks=build_banks(os.path.join(root, "banks")))


def _setup(corpus, fe_alg, T):
    from distortion_banks import case_cfg
    from helpers import fill_state_dict
    from pase_b200.batch import DeviceBatcher, WavPool
    from pase_b200.distortions import config_distortions
    from test_train_step import RECIPES, make_model
    _, wcfg, _ = RECIPES["pase+"]
    model = make_model("pase+")
    model.load_state_dict(fill_state_dict(model.state_dict(), 5))
    model.frontend.precision = "3xf16"
    model = model.cuda().train()
    # the reference trainer's layout for --fe_opt <fe_alg> --min_opt radam
    groups = [{"params": list(model.frontend.parameters()), "algorithm": fe_alg}]
    groups += [{"params": list(w.parameters()), "algorithm": "radam"} for w in
               list(model.classification_workers) + list(model.regression_workers)]
    engine = FlatAdam(groups, lr=5e-4).bind_encoder(model.frontend)
    wavs = WavPool(corpus["data_root"], corpus["cfg"], "train", placement="cuda")
    dist = config_distortions(device="cuda", **case_cfg("pase_plus", corpus["banks"])[0])
    batcher = DeviceBatcher.from_train_opts(
        wcfg, T, 160, wavs, random_scale=True, distortions=dist,
        trans_cache=os.path.join(corpus["root"], "cache_pase+"))
    return model, engine, batcher


@pytest.mark.parametrize("fe_alg", ["adam", "radam"])
def test_graphed_train_step_with_radam_equals_eager(fe_alg, corpus):
    """8 steps: 3 eager warm-up calls, the capture, 4 replays.  RAdam's rho crosses 5 at step 6,
    inside the replays; the lr schedule changes every group before every call."""
    import random
    from pase_b200 import functional as Fn
    from pase_b200.batch import WavPool
    from pase_b200.graph import GraphedTrainStep
    from pase_b200.pase import total_loss
    from test_train_step_gpu import _batches, _compare, _poly, _seed
    steps, B, T = 8, 4, 16000
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        batches = _batches(len(WavPool(corpus["data_root"], corpus["cfg"], "train",
                                       placement="cpu")), B, steps, 11)
        model, engine, batcher = _setup(corpus, fe_alg, T)
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
        gmodel, gengine, gbatcher = _setup(corpus, fe_alg, T)
        step = GraphedTrainStep(gmodel, gengine, gbatcher, B)
        _seed(3)
        for k, (new_epoch, idx) in enumerate(batches):
            if new_epoch:
                gbatcher.reset()
            _poly(gengine, k, steps)
            step(idx)
        assert step.graph is not None and step.calls == steps and step.warmup < 5
        got = step.losses()
        torch.cuda.synchronize()
        for n in eager:
            assert got[n] == eager[n], (n, got[n], eager[n])
        _compare(engine, gengine)
        assert float(gengine.steps[0]) == steps
    finally:
        Fn.set_precision(prev)
        random.seed()


# ---------------------------------------------------------------- peer_dp on two GPUs

def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _peer_worker(rank, world, port, out):
    """FlatAdam(peer_dp=True) with an Adam and two RAdam groups over seven steps, against the
    float64 restatement on the all-gathered mean gradient."""
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    gen = torch.Generator().manual_seed(4)
    shapes = [[(33, 7), (7,)], [(129,), (5, 5)], [(1001,)]]
    params = [[torch.nn.Parameter(torch.randn(s, generator=gen).to(dev)) for s in grp]
              for grp in shapes]
    groups = [{"params": params[0], "algorithm": "adam", "lr": 1e-3},
              {"params": params[1], "algorithm": "radam", "lr": 2e-3, "weight_decay": 1e-2},
              {"params": params[2], "algorithm": "radam", "lr": 5e-3, "betas": (0.8, 0.99)}]
    opt = FlatAdam(groups, peer_dp=True)
    assert opt._peer is not None
    rows = []
    for gi, ((a, b), g) in enumerate(zip(opt._ranges, opt.param_groups)):
        rows.append(dict(start=a, end=b, lr=_f32(g["lr"]), b1=_f32(g["betas"][0]),
                         b2=_f32(g["betas"][1]), eps=_f32(g["eps"]), wd=_f32(g["weight_decay"]),
                         algo=1.0 if g["algorithm"] == "radam" else 0.0, si=gi))
    p_ref = opt.flat_param.clone()
    m_ref = torch.zeros_like(p_ref)
    v_ref = torch.zeros_like(p_ref)
    ggen = torch.Generator().manual_seed(100 + rank)
    for it in range(1, 8):
        for grp in params:
            for p in grp:
                p.grad = torch.randn(p.shape, generator=ggen).to(dev) * 1e-2
        opt.pack_grads()
        torch.cuda.synchronize()
        gathered = [torch.empty_like(opt.flat_grad) for _ in range(world)]
        dist.all_gather(gathered, opt.flat_grad.clone())
        mean = sum(t.double() for t in gathered) / world
        want = restate(rows, p_ref, mean, m_ref, v_ref, [float(it)] * 3)
        opt.step()
        torch.cuda.synchronize()
        err = (opt.flat_param.double() - want[0]).abs()
        bound = 3e-7 * want[0].abs() + 1e-5 * (want[0] - p_ref.double()).abs() + 1e-7 * 5e-3
        assert bool((err <= bound).all()), (rank, it, float(err.max()))
        p_ref = opt.flat_param.clone()
        m_ref, v_ref = want[1].float(), want[2].float()
        both = [torch.empty_like(opt.flat_param) for _ in range(world)]
        dist.all_gather(both, opt.flat_param.clone())
        assert torch.equal(both[0], both[1])
    opt.consolidate_state()
    sd = opt.state_dict()
    assert sd["state"][2]["step"] == 7 and "amsgrad" not in sd["param_groups"][1]
    if rank == 0:
        open(os.path.join(out, "ok"), "w").write("ok")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_peer_dp_radam_two_gpus(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_peer_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert os.path.exists(tmp_path / "ok")
