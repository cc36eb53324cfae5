"""The captured validation pass on the GPU: GraphedEvalStep equals the eager pass (batcher ->
model.eval() forward under no_grad -> each worker's unweighted loss and their sum) bit for bit,
with fused regression heads on and off; it sees the weights and BatchNorm statistics training
steps wrote and changes none of them; a replayed batch launches nothing from Python and copies
one plan in and nothing out; the fused heads take no memory under no_grad; the loss-only
epilogue gives the loss of the full one.
"""
import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode
from torch.utils._pytree import tree_flatten

from pase_b200 import _lib, ops
from pase_b200 import functional as Fn
from pase_b200.batch import WavPool
from pase_b200.graph import GraphedEvalStep, GraphedTrainStep
from pase_b200.pase import eval_losses
from test_tc_gemm_gpu import R, _operands
from test_train_step_gpu import _batches, _seed, _setup, _triple
from test_train_step_gpu import corpus  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


def _eager_pass(model, batcher, batches, rng):
    """The reference _eval loop body: per batch, every worker's loss and the total."""
    rows = []
    for new_epoch, idx in batches:
        if new_epoch:
            batcher.reset()
        with torch.no_grad():
            _, _, preds, labels = model(batcher(idx, rng))
            tot, losses = eval_losses(model, preds, labels)
        rows.append(dict({n: v.reshape(()).clone() for n, v in losses.items()}, total=tot))
    torch.cuda.synchronize()
    return {n: [float(r[n]) for r in rows] for n in rows[0]}


def _graphed_pass(ev, batcher, batches, rng):
    for new_epoch, idx in batches:
        if new_epoch:
            batcher.reset()
        ev(idx, rng)
    return ev.losses()


def _assert_equal(got, ref):
    assert list(got) == list(ref)
    for n in ref:
        assert got[n] == ref[n], (n, got[n], ref[n])


def _n(corpus):
    return len(WavPool(corpus["data_root"], corpus["cfg"], "train", placement="cpu"))


CASES = [("pase+", "3xf16", 4, 16000, False, False), ("pase+", "3xf16", 4, 16000, False, True),
         ("pase+", "bf16", 4, 16000, False, False), ("pase+", "bf16", 4, 16000, False, True),
         ("pase", "fp32", 4, 16000, True, False), ("pase+", "3xf16", 32, 32000, False, True)]


@pytest.mark.parametrize("recipe,precision,B,T,triple,fuse", CASES)
def test_graphed_pass_equals_the_eager_pass(recipe, precision, B, T, triple, fuse, corpus):
    nb = 6
    prev = Fn.PRECISION
    Fn.set_precision(precision)
    try:
        batches = _batches(_n(corpus), B, nb, 17)
        model, _, batcher = _setup(corpus, recipe, T, precision)
        model.fuse_regression_loss = fuse
        model.eval()
        # eager: the global generators (SPCMinion draws from `random`); the triple seeded alike
        # draws the same streams
        _seed(4)
        eager = _eager_pass(model, batcher, batches, None)
        gmodel, _, gbatcher = _setup(corpus, recipe, T, precision)
        gmodel.fuse_regression_loss = fuse
        gmodel.eval()
        ev = GraphedEvalStep(gmodel, gbatcher, B, max_batches=nb)
        rng = None
        if triple:
            rng = _triple(4)
        else:
            _seed(4)
        got = _graphed_pass(ev, gbatcher, batches, rng)
        assert ev.graph is not None and ev.calls == nb
        _assert_equal(got, eager)
        if recipe == "pase":
            assert len(ev.planner.spc) == 1 and "spc" in got
    finally:
        Fn.set_precision(prev)


def _state(model):
    return {k: v.clone() for k, v in model.state_dict().items()}


def test_passes_between_training_replays(corpus):
    """train replays, eval pass, train replays, eval pass: each pass equals an eager pass on a
    second batcher at the same point, with the same draws; the passes change no parameter,
    running statistic or step counter."""
    B, T, nb = 4, 16000, 5
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        model, engine, tbatcher = _setup(corpus, "pase+", T, "3xf16")
        model.fuse_regression_loss = True
        _, _, vbatcher = _setup(corpus, "pase+", T, "3xf16")
        _, _, ebatcher = _setup(corpus, "pase+", T, "3xf16")
        step = GraphedTrainStep(model, engine, tbatcher, B)
        ev = GraphedEvalStep(model, vbatcher, B, max_batches=nb)
        train = _batches(_n(corpus), B, 8, 21)
        _seed(6)
        for p, (lo, hi) in enumerate(((0, 5), (5, 8))):
            model.train()
            for _, idx in train[lo:hi]:
                step(idx)
            model.eval()
            # no synchronise: the pass is ordered after the steps on the device
            before = _state(model)
            batches = _batches(_n(corpus), B, nb, 30 + p)
            vbatcher.reset()
            got = _graphed_pass(ev, vbatcher, batches, _triple(40 + p))
            ev.reset()
            after = _state(model)
            for k, v in before.items():
                assert torch.equal(after[k], v), k
            ebatcher.reset()
            ref = _eager_pass(model, ebatcher, batches, _triple(40 + p))
            _assert_equal(got, ref)
        assert step.graph is not None and ev.graph is not None
    finally:
        Fn.set_precision(prev)


class _Copies(TorchDispatchMode):
    """Counts host-to-device and device-to-host tensor copies, and every torch operation that
    touches a CUDA tensor, issued from Python inside the block.  (Counted at the dispatcher
    rather than with torch.profiler: a profiler session opened after earlier sessions in the
    same process can miss the first copy of the block.)"""

    def __init__(self):
        super().__init__()
        self.h2d = self.d2h = 0
        self.cuda_ops = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        flat = [t for t in tree_flatten((args, kwargs))[0] if isinstance(t, torch.Tensor)]
        if any(t.is_cuda for t in flat):
            self.cuda_ops.append(func)
        if func is torch.ops.aten.copy_.default:
            dst, src = args[0], args[1]
            self.h2d += int(dst.is_cuda and not src.is_cuda)
            self.d2h += int(src.is_cuda and not dst.is_cuda)
        return func(*args, **kwargs)


def test_replay_launches_copies_and_refusals(corpus):
    B, T = 4, 16000
    model, _, batcher = _setup(corpus, "pase", T, "3xf16")
    ev = GraphedEvalStep(model, batcher, B, max_batches=4, warmup=1)
    batches = _batches(len(batcher.wavs), B, 4, 2)
    with pytest.raises(ValueError, match="train mode"):
        ev(batches[0][1])
    model.eval()
    for _, idx in batches[:2]:                   # warm-up, capture + replay
        ev(idx)
    with pytest.raises(ValueError, match="batch of 3"):
        ev(batches[2][1][:3])
    torch.cuda.synchronize()
    n0 = ops.launch_count
    with _Copies() as c:
        ev(batches[2][1])
        torch.cuda.synchronize()
    assert ops.launch_count == n0
    # the plan upload is the only torch operation on a CUDA tensor: the rest is one replay
    assert c.cuda_ops == [torch.ops.aten.copy_.default], c.cuda_ops
    assert (c.h2d, c.d2h) == (1, 0)
    ev(batches[3][1])
    with pytest.raises(RuntimeError, match="reset"):
        ev(batches[0][1])
    with _Copies() as c:
        losses = ev.losses()
    assert (c.h2d, c.d2h) == (0, 1)
    assert list(losses) == ["spc", "mi", "cmi", "cchunk", "lps", "mfcc", "prosody", "total"]
    assert all(len(v) == 4 and all(x == x for x in v) for v in losses.values())
    ev.reset()
    batcher.reset()                              # the batcher's own epoch bookkeeping
    ev(batches[0][1])
    assert all(len(v) == 1 for v in ev.losses().values())


def test_fused_heads_take_no_memory_without_grad(corpus):
    B, T = 4, 16000
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        model, _, batcher = _setup(corpus, "pase+", T, "3xf16")
        model.fuse_regression_loss = True
        model.eval()
        batch = batcher(_batches(len(batcher.wavs), B, 1, 3)[0][1])
        pool = {k: len(v) for k, v in Fn._FusedLinearCtxMSE._buffers.items()}
        mem = []
        for i in range(22):
            with torch.no_grad():
                _, _, preds, labels = model(batch)
                tot, _ = eval_losses(model, preds, labels)
                assert any(hasattr(p, "_pase_fused_loss") for p in preds.values())
            del preds, labels, tot
            torch.cuda.synchronize()
            if i >= 2:                      # after the plans and constants are built
                mem.append(torch.cuda.memory_allocated())
        # no growth: every forward ends in the band of the first two (which alternate by a few
        # hundred KB as the last output is replaced); one residual pair here is 35 MB
        assert min(mem[:2]) <= min(mem) and max(mem) <= max(mem[:2]), mem
        assert max(mem) - min(mem) < 4 << 20, mem
        assert {k: len(v) for k, v in Fn._FusedLinearCtxMSE._buffers.items()} == pool
    finally:
        Fn.set_precision(prev)


def test_loss_only_epilogue_equals_the_full_one():
    """Same operands through pase_tc_gemm_nt_ctxmse with and without the residual pair: the
    fp64 losses agree to 1e-14 and are equal in fp32 (the criterion of
    test_tc_gemm_nt_ctxmse_reproducible)."""
    Bn, F, T, r, K = 4, 40, 700, 3, 256
    M, N, Rr, ldr = Bn * T, F * r, 256, 128
    a_rows = M + 3
    A, W = R(a_rows * Rr, seed=131), R(N * K, seed=132, scale=0.1)
    (Ah, Al), (Bh, Bl) = _operands(A, 3), _operands(W, 3, weights=True)
    d = [t.cuda() for t in (Ah, Al, Bh, Bl)]
    bias, label = R(N, seed=133).cuda(), R(Bn * F * T, seed=134).cuda()
    scale = torch.tensor([1.0 / 64, 64.0]).cuda()
    rh, rl = (torch.zeros(M * ldr, dtype=torch.float16, device="cuda") for _ in range(2))
    full = torch.zeros(1, dtype=torch.float64, device="cuda")
    db = torch.zeros(N, dtype=torch.float64, device="cuda")
    _lib.call("pase_tc_gemm_nt_ctxmse", d[0], d[1], a_rows, Rr, d[2], d[3], K, rh, rl, ldr,
              M, N, K, bias, label, Bn, F, T, r, scale, full, db)
    only = torch.zeros(1, dtype=torch.float64, device="cuda")
    _lib.call("pase_tc_gemm_nt_ctxmse", d[0], d[1], a_rows, Rr, d[2], d[3], K, None, None, ldr,
              M, N, K, bias, label, Bn, F, T, r, None, only, None)
    torch.cuda.synchronize()
    assert float(full) > 0
    assert abs(float(full) - float(only)) <= 1e-14 * abs(float(full))
    assert torch.equal(full.float(), only.float())
    # a half-given residual is refused
    with pytest.raises(RuntimeError, match="null pointer"):
        _lib.call("pase_tc_gemm_nt_ctxmse", d[0], d[1], a_rows, Rr, d[2], d[3], K, rh, None, ldr,
                  M, N, K, bias, label, Bn, F, T, r, scale, only, db)
