"""Data parallelism on real GPUs (2 ranks, NCCL over NVLink): the flat-buffer all-reduce
averages the per-rank gradients, and the pipelined step (all-reduce hidden behind the tail
of backward, three CUDA graphs) equals the plain eager step.  Needs >= 2 GPUs (skips
otherwise):
    python -m pytest tests/test_dp_nccl_gpu.py -m gpu
"""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512, "denseskips": True,
             "norm_out": True, "rnn_pool": True, "rnn_layers": 1}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    import torch.distributed as dist
    from pase_b200 import wf_builder
    from pase_b200.optim import FlatAdam
    from pase_b200.graph import PipelinedDPStep
    from pase_b200.dp import broadcast_parameters_and_buffers
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    side = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(side)
    B, T, split = 4, 8000, 3
    loss_fn = lambda y: y.square().mean()
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(100 + rank)).to(dev)

    def build(seed):
        torch.manual_seed(seed + rank)                  # replicas start different ...
        m = wf_builder(dict(PASE_PLUS)).to(dev).train()
        broadcast_parameters_and_buffers(m)             # ... and are aligned to rank 0
        params, n_lower = PipelinedDPStep.order_params(m, split)
        opt = FlatAdam(params, lr=1e-3).bind_encoder(m)
        return m, opt, n_lower

    # (1) the collective: reduced flat gradient == mean over ranks of the local gradients
    m, opt, n_lower = build(0)
    loss_fn(m(x)).backward()
    local = opt.flat_grad.clone()
    gathered = [torch.empty_like(local) for _ in range(world)]
    dist.all_gather(gathered, local)
    opt.reduce_grads()
    mean = sum(gathered) / world
    assert torch.allclose(opt.flat_grad, mean, rtol=1e-5, atol=1e-8 + 1e-6 * float(mean.abs().max()))
    assert float((gathered[0] - gathered[1]).abs().max()) > 0      # the shards really differ

    # (2) pipelined graphs == eager.  Adam turns ANY gradient into a +-lr step, so parameters
    # are a poor witness (noise-level gradients flip signs between two runs); the reduced flat
    # gradient is compared instead, with lr = 0 so that every step sees the same weights.
    def build0(seed):
        m, _, n_lower = build(seed)
        params, n_lower = PipelinedDPStep.order_params(m, split)
        m.grad_sink = None
        return m, FlatAdam(params, lr=0.0).bind_encoder(m), n_lower
    ma, oa, _ = build0(1)
    mb, ob, n_lower = build0(1)
    for (ka, pa), (kb, pb) in zip(ma.named_parameters(), mb.named_parameters()):
        assert torch.equal(pa, pb), ka
    loss_fn(ma(x)).backward()
    oa.reduce_grads()
    oa.step()
    ga = oa.flat_grad.clone()
    # 1 eager warm-up step inside the constructor (lazy tables / plans must exist before the
    # capture) + 2 graph replays = 3 optimizer steps
    pipe = PipelinedDPStep(mb, ob, loss_fn, (B, 1, T), dev, split=split, n_lower=n_lower,
                           stream=side, resident=True, warmup=1, x_init=x.cpu().pin_memory())
    worst = 0.0
    for _ in range(2):
        ob.flat_grad.zero_()                       # a stale buffer must not pass the check
        pipe.step()
        torch.cuda.synchronize()
        gb = ob.flat_grad
        # two model instances see BatchNorm statistics that differ in the last bit (fp64
        # atomics), which now and then flips one PReLU gate: at B=4, T=8000 that moves whole
        # gradient rows by ~1e-3 of the norm.  A stale, unreduced or misplaced bucket would be
        # an O(1) error: relative L2 of the whole flat gradient + a loose elementwise bound.
        err = float((ga - gb).norm() / ga.norm())
        worst = max(worst, err)
        assert err <= 1.5e-2, err
        assert float((ga - gb).abs().max()) <= 5e-2 * float(ga.abs().max())
    assert float(ob.steps[0]) == 3.0 and float(oa.steps[0]) == 1.0
    # every rank holds the same parameters afterwards
    flat = ob.flat_param.clone()
    both = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(both, flat)
    assert torch.equal(both[0], both[1])
    if rank == 0:
        open(os.path.join(out, "ok"), "w").write(
            "pipelined vs eager reduced gradient: worst relative L2 = %.3e\n" % worst)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_flat_allreduce_and_pipelined_step_two_gpus(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert os.path.exists(tmp_path / "ok")
    print(open(tmp_path / "ok").read())


def _peer_worker(rank, world, port, out):
    """pase_adam_flat_dp (reduce-scatter + Adam + all-gather over CUDA-IPC peer memory, one
    kernel) against torch arithmetic on the all-gathered gradients; then the captured step."""
    import torch.distributed as dist
    from pase_b200 import wf_builder
    from pase_b200.optim import FlatAdam
    from pase_b200.graph import GraphedEncoderStep
    from pase_b200.dp import broadcast_parameters_and_buffers
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    side = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(side)
    B, T = 4, 8000
    loss_fn = lambda y: y.square().mean()
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(200 + rank)).to(dev)
    torch.manual_seed(7 + rank)
    m = wf_builder(dict(PASE_PLUS)).to(dev).train()
    broadcast_parameters_and_buffers(m)
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    opt = FlatAdam(list(m.parameters()), lr=lr, betas=(b1, b2), eps=eps, peer_dp=True).bind_encoder(m)
    assert opt._peer is not None and opt._peer.world == world
    lo, hi = opt.shard_range()
    p_ref = opt.flat_param.double().clone()
    m_ref = torch.zeros_like(p_ref)
    v_ref = torch.zeros_like(p_ref)
    worst = 0.0
    for it in range(1, 4):
        opt.zero_grad(set_to_none=True)
        loss_fn(m(x)).backward()
        opt.pack_grads()
        torch.cuda.synchronize()
        local = opt.flat_grad.clone()
        gathered = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(gathered, local)
        g = sum(t.double() for t in gathered) / world
        assert float((gathered[0] - gathered[1]).abs().max()) > 0
        p_old = opt.flat_param.double().clone()
        opt.step()
        torch.cuda.synchronize()
        # reference Adam on the mean gradient (torch.optim.Adam semantics, float64)
        m_ref = b1 * m_ref + (1 - b1) * g
        v_ref = b2 * v_ref + (1 - b2) * g * g
        denom = v_ref.sqrt() / (1 - b2 ** it) ** 0.5 + eps
        p_ref = p_ref - (lr / (1 - b1 ** it)) * m_ref / denom
        # padding elements between parameters are never touched by the kernel
        live = torch.zeros(opt.n, dtype=torch.bool, device=dev)
        for p, o in zip(opt._plist, opt._offsets):
            live[o:o + p.numel()] = True
        # the step is ~lr per element; the sinc cut-offs (~5e3 Hz) are coarser than that in
        # fp32 (ulp 4.9e-4): their update is whatever rounding leaves of it
        diff = ((opt.flat_param.double() - p_ref).abs() - 2.4e-7 * p_ref.abs()).clamp_min(0) * live
        dp = diff.max()
        worst = max(worst, float(dp) / lr)
        if float(dp) > 2e-3 * lr:
            j = int(diff.argmax())
            name = [k for (k, p), o in zip(m.named_parameters(), opt._offsets)
                    if o <= j < o + p.numel()]
            nbad = int((diff > 2e-3 * lr).sum())
            raise AssertionError(
                "step %d rank %d: |dp| %.3e at flat index %d (%s, shard of rank %d), %d elements "
                "off; g0 %.6e g1 %.6e mean %.6e  p_old %.8e p_kernel %.8e p_ref %.8e"
                % (it, rank, float(dp), j, name, 0 if j < hi and rank == 0 or j < lo else 1, nbad,
                   float(gathered[0][j]), float(gathered[1][j]), float(g[j]), float(p_old[j]),
                   float(opt.flat_param[j]), float(p_ref[j])))
        assert torch.allclose(opt.exp_avg[lo:hi].double()[live[lo:hi]], m_ref[lo:hi][live[lo:hi]],
                              rtol=1e-5, atol=1e-9)
        # every rank holds the same parameters
        both = [torch.empty_like(opt.flat_param) for _ in range(world)]
        dist.all_gather(both, opt.flat_param.clone())
        assert torch.equal(both[0], both[1])
        p_ref = opt.flat_param.double().clone()      # next step starts from the fp32 state
    opt.consolidate_state()
    live_idx = live.nonzero().squeeze(1)
    assert torch.allclose(opt.exp_avg.double()[live_idx], m_ref[live_idx], rtol=1e-5, atol=1e-9)
    assert torch.allclose(opt.exp_avg_sq.double()[live_idx], v_ref[live_idx], rtol=1e-5, atol=1e-12)
    # the whole step (forward, backward, fused DP update) as ONE CUDA graph, 3 replays
    gs = GraphedEncoderStep(m, opt, loss_fn, (B, 1, T), dev, stream=side, resident=True,
                            warmup=1, x_init=x.cpu().pin_memory())
    for _ in range(3):
        gs.step()
    torch.cuda.synchronize()
    both = [torch.empty_like(opt.flat_param) for _ in range(world)]
    dist.all_gather(both, opt.flat_param.clone())
    assert torch.equal(both[0], both[1]) and bool(torch.isfinite(both[0]).all())
    assert float(opt.steps[0]) == 3 + 1 + 3
    if rank == 0:
        open(os.path.join(out, "ok_peer"), "w").write(
            "pase_adam_flat_dp vs float64 Adam on the gathered gradients: worst |dp| = %.2e lr\n" % worst)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_peer_memory_dp_update_two_gpus(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_peer_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert os.path.exists(tmp_path / "ok_peer")
    print(open(tmp_path / "ok_peer").read())
