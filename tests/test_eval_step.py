"""The validation pass (reference trainer ``_eval``, trainer.py:282-337), CPU side: the native
eager pass equals what the unmodified reference computed (tests/golden/eval.pt, written by
tests/golden/make_eval_golden.py), the fused regression head under ``no_grad`` takes no
residual buffer, the loss-only form of the fused epilogue's spec gives the loss of the full
form, and GraphedEvalStep refuses what it cannot run.  CUDA kernels are replaced by their torch
specs (tests/emul/); tests/test_eval_step_gpu.py
covers the kernels.
"""
import copy
import json
import os
import random

import pytest
import torch

import emul
from helpers import GOLDEN, resolve_cfg, seeded_randn
from pase_b200 import encoder as enc
from pase_b200 import functional as Fn
from pase_b200 import ops
from pase_b200.frontend import WaveFe
from pase_b200.graph import GraphedEvalStep
from pase_b200.pase import eval_losses, pase as native_pase
from pase_b200.utils import parse_workers
from test_train_step import _cpu_batcher, build_corpus, make_model


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)

    def encode_cpu(self, x):
        self._sinc_consts(x.device)
        plan = self._plan(x.shape[0], x.shape[2], x.device)
        named = list(self.named_parameters())
        return enc._EncoderFn.apply(x.contiguous().float(), self, plan, self.training,
                                    tuple(n for n, _ in named), *[p for _, p in named])
    monkeypatch.setattr(WaveFe, "encode", encode_cpu)
    yield


def _eval_batch(B, T, Tq, wcfg, seed):
    """make_eval_golden.eval_batch: the four waveforms and one label per regression worker."""
    batch = {k: seeded_randn((B, 1, T), seed + i, 0.5)
             for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
    for i, w in enumerate(wcfg["regr"]):
        if w["name"] != "cchunk":
            batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)
    return batch


def _eager_pass(model, batches):
    """The reference _eval loop body on the native model: running_loss per worker and total."""
    running = {}
    with torch.no_grad():
        for batch in batches:
            _, _, preds, labels = model(batch)
            tot, losses = eval_losses(model, preds, labels)
            for k, v in list(losses.items()) + [("total", tot)]:
                running.setdefault(k, []).append(float(v))
    return running


@pytest.mark.parametrize("fuse", [False, True])
def test_eager_pass_matches_the_reference_eval(fuse, emulated):
    gold = torch.load(os.path.join(GOLDEN, "eval.pt"), map_location="cpu")
    meta = json.loads(gold["meta"])
    B, T, Tq, seed = meta["B"], meta["T"], meta["Tq"], meta["seed"]
    wcfg = meta["workers"]
    model = native_pase(frontend_cfg=resolve_cfg(meta["fe_cfg"]),
                        minions_cfg=parse_workers(copy.deepcopy(wcfg)))
    state = {k[len("state/"):]: v for k, v in gold.items() if k.startswith("state/")}
    assert sorted(state) == sorted(model.state_dict())
    model.load_state_dict(state)
    model.fuse_regression_loss = fuse
    model.eval()
    batches = [_eval_batch(B, T, Tq, wcfg, seed + 1000 + 200 * i)
               for i in range(meta["batches"])]
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        random.seed(seed + 50)
        got = _eager_pass(model, batches)
    finally:
        Fn.set_precision(prev)
    names = json.loads(gold["names"])
    assert list(got) == names                     # running_loss's key order
    for k in names:
        ref = gold["loss/" + k].tolist()
        assert len(got[k]) == len(ref) == meta["batches"]
        for i, (a, b) in enumerate(zip(got[k], ref)):
            assert abs(a - b) <= 2e-4 * max(abs(b), 1e-3), (k, i, a, b)


def _fused_operands(seed=3):
    B, T, F, r, K = 2, 40, 12, 3, 64
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(B * T, K, generator=gen)
    w = torch.randn(F * r, K, 1, generator=gen) * 0.1
    b = torch.randn(F * r, generator=gen)
    label = torch.randn(B, F, T, generator=gen)
    return h, w, b, label, F, r


def test_fused_head_without_grad_takes_no_residual_buffer(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    h, w, b, label, F, r = _fused_operands()
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        assert Fn.fused_head_ok(h.shape[1], h.shape[1])
        before = {k: len(v) for k, v in Fn._FusedLinearCtxMSE._buffers.items()}
        w, b = w.requires_grad_(True), b.requires_grad_(True)
        with torch.no_grad():
            losses = [Fn.fused_linear_ctx_mse(h, w, b, label, F, r) for _ in range(10)]
        # nothing requires grad: no backward will run either
        losses += [Fn.fused_linear_ctx_mse(h, w.detach(), b.detach(), label, F, r)]
        after = {k: len(v) for k, v in Fn._FusedLinearCtxMSE._buffers.items()}
        assert after == before
        assert all(torch.equal(x, losses[0]) for x in losses)
        # with a gradient to come the pool serves the pair, and backward releases it
        loss = Fn.fused_linear_ctx_mse(h, w, b, label, F, r)
        loss.backward()
        assert torch.equal(loss.detach(), losses[0])
        assert all(not e["busy"] for v in Fn._FusedLinearCtxMSE._buffers.values() for e in v)
    finally:
        Fn.set_precision(prev)


def test_emulated_loss_only_spec_equals_the_full_spec():
    h, w, b, label, F, r = _fused_operands(5)
    rows, K = h.shape
    N = F * r
    ldr = 128
    hi, lo = torch.zeros(rows * K, dtype=torch.float16), torch.zeros(rows * K, dtype=torch.float16)
    whi, wlo = torch.zeros(N * K, dtype=torch.float16), torch.zeros(N * K, dtype=torch.float16)
    emul.call("pase_split_f16", h.reshape(-1), hi, lo, rows * K, None, None)
    emul.call("pase_split_f16", w.reshape(-1), whi, wlo, N * K, None, None)
    scale = torch.tensor([1.0 / 64, 64.0])
    full = torch.zeros(1, dtype=torch.float64)
    db = torch.zeros(N, dtype=torch.float64)
    rh, rl = (torch.zeros(rows * ldr, dtype=torch.float16) for _ in range(2))
    common = (hi, lo, rows, K, whi, wlo, K)
    tail = (rows, N, K, b, label.reshape(-1), label.shape[0], F, label.shape[2], r)
    emul.call("pase_tc_gemm_nt_ctxmse", *common, rh, rl, ldr, *tail, scale, full, db)
    only = torch.zeros(1, dtype=torch.float64)
    emul.call("pase_tc_gemm_nt_ctxmse", *common, None, None, ldr, *tail, None, only, None)
    assert float(full) > 0 and torch.equal(only, full)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("eval_corpus"))
    return build_corpus(root, 24, 9000, 20000)


def test_refusals(corpus):
    model = make_model("pase").eval()
    batcher = _cpu_batcher(corpus, "pase", 8000)
    with pytest.raises(ValueError, match="warmup"):
        GraphedEvalStep(model, batcher, 4, warmup=0)
    with pytest.raises(ValueError, match="batch_size"):
        GraphedEvalStep(model, batcher, 0)
    # 4000 samples -> T' = 25 frames: SPC's range(22, 4) for the current frame is empty
    with pytest.raises(ValueError, match="no current frame"):
        GraphedEvalStep(model, _cpu_batcher(corpus, "pase", 4000), 4)
    with pytest.raises(ValueError, match="CUDA"):
        GraphedEvalStep(model, batcher, 4)
