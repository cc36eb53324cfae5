"""CUDA-graph captured training step == eager step (same kernels, same numerics)."""
import pytest
import torch

from helpers import resolve_cfg, fill_state_dict, seeded_randn, rel_l2
from pase_b200.frontend import WaveFe
from pase_b200.graph import GraphedEncoderStep

pytestmark = pytest.mark.gpu


def _model(seed):
    cfg = resolve_cfg("cfg/frontend/PASE+.cfg")
    m = WaveFe(**cfg)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed))
    return m.cuda().train()


@pytest.mark.parametrize("split", [False, True])
def test_graphed_step_matches_eager(split):
    """split=True: the data-parallel form -- [forward, backward, pack gradients into the flat
    buffer] and [optimizer] are two graphs with an eager hook (the all-reduce; a no-op
    collective in a single process) between their replays."""
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    try:
        x = seeded_randn((4, 1, 6400), 5, 0.5)
        cot = seeded_randn((4, 256, 40), 6).cuda()
        loss_fn = lambda y: (y * cot).mean() + y.abs().mean()     # not invariant under norm_out
        # eager: two Adam steps
        me = _model(3)
        # SGD: linear in the gradients (Adam would turn the fp-noise gradients of the
        # analytically-zero conv biases into +-lr steps of random sign)
        oe = torch.optim.SGD(me.parameters(), lr=1e-2, momentum=0.9, foreach=True)
        eager_losses = []
        for _ in range(3 + 2):                       # same number of updates as warm-up + replays
            oe.zero_grad(set_to_none=True)
            l = loss_fn(me(x.cuda()))
            l.backward()
            oe.step()
            eager_losses.append(float(l))
        # graphed: 3 warm-up updates inside the constructor, capture (1 update), then 1 replay
        mg = _model(3)
        og = torch.optim.SGD(mg.parameters(), lr=1e-2, momentum=0.9, foreach=True)
        kw = {}
        if split:
            from pase_b200.dp import FlatGradAllReducer
            red = FlatGradAllReducer(list(mg.parameters()), attach=False)
            kw = dict(post_backward=red.pack, between=red.all_reduce)
        gs = GraphedEncoderStep(mg, og, loss_fn, (4, 1, 6400), "cuda", stream=side, warmup=3,
                                x_init=x, **kw)
        assert (gs.graph_b is not None) == split
        # the capture itself does not execute; replays do
        l1 = gs.step()
        l2 = gs.step()
        # the same kernels in the same order, and no sum depends on thread scheduling: the
        # replayed steps reproduce the eager steps bit for bit
        assert l1 == eager_losses[3] and l2 == eager_losses[4], (l1, l2, eager_losses[3:])
        assert abs(eager_losses[4] - eager_losses[3]) > 1e-3 * abs(eager_losses[3])   # loss moves
        for (k, pe), (_, pg) in zip(me.named_parameters(), mg.named_parameters()):
            assert torch.equal(pg.detach(), pe.detach()), \
                (k, rel_l2(pg.detach().cpu(), pe.detach().cpu()))
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())
