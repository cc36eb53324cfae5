"""Worker heads + pase wrapper + summed multi-task loss: host logic on CPU with emulated
kernels against golden vectors produced by the unmodified reference."""
import random

import pytest
import torch

import emul
from helpers import load_golden, resolve_cfg, fill_state_dict, seeded_randn, assert_close, \
    check_grads
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import WaveFe
from pase_b200.pase import pase as native_pase, total_loss
from pase_b200.utils import parse_workers


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)

    def encode_cpu(self, x):
        self._sinc_consts(x.device)
        plan = self._plan(x.shape[0], x.shape[2], x.device)
        named = list(self.named_parameters())
        names = tuple(n for n, _ in named)
        return enc._EncoderFn.apply(x.contiguous().float(), self, plan, self.training, names,
                                    *[p for _, p in named])
    monkeypatch.setattr(WaveFe, "encode", encode_cpu)
    yield


def build_case(name, device="cpu"):
    gold, meta = load_golden(name)
    fe_cfg, wcfg = resolve_cfg(meta["fe_cfg"]), meta["workers"]
    model = native_pase(frontend_cfg=fe_cfg, minions_cfg=parse_workers(wcfg))
    model.load_state_dict(fill_state_dict(model.state_dict(), meta["seed"]))
    model = model.to(device).train()
    B, T, Tq, seed = meta["B"], meta["T"], meta["Tq"], meta["seed"]
    batch = {k: seeded_randn((B, 1, T), seed + 10 + i, 0.5)
             for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
    for i, w in enumerate(wcfg["regr"]):
        if w["name"] != "cchunk":
            batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)
    return gold, meta, model, batch


def check_case(gold, meta, model, batch, device, rtol=1e-4, atol=1e-5):
    random.seed(meta["seed"])
    h, chunk, preds, labels = model(batch, 1, device)
    assert len(h) == 3 and tuple(chunk.shape) == tuple(gold["chunk"].shape)
    assert_close(chunk, gold["chunk"], rtol, atol, "chunk")
    tot, losses = total_loss(model, preds, labels)
    for k, v in losses.items():
        assert_close(v, gold["loss/" + k], 2e-4, 1e-6, "loss " + k)
    assert_close(tot, gold["total"], 2e-4, 1e-6, "total")
    for k, v in gold.items():
        if k.startswith("pred/"):
            assert tuple(preds[k[5:]].shape) == tuple(v.shape), k
            assert_close(preds[k[5:]], v, 10 * rtol, 10 * atol, k)
    tot.backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    assert all(g is not None for g in grads.values())
    dec = ["regression_workers.%d." % i for i, w in enumerate(meta["workers"]["regr"])
           if w.get("type") == "decoder"]
    assert check_grads(grads, gold, 2e-3, 2e-4, l2_keys=dec) > 20


def _workers_case(name, precision):
    # the heads' default precision keeps the bare case name as its test id
    return pytest.param(name, precision, id=name if precision == "3xf16" else
                        "%s-%s" % (name, precision))


# tf32 and bf16 miss the fp32 bars by their operand formats
@pytest.mark.parametrize("name,precision", [
    _workers_case(n, p) for n in ("pase_mini_workers_1600", "pase_plus_workers_3200")
    for p in ("3xf16", "3xtf32", "fp32")])
def test_pase_workers_host_logic(name, precision, emulated, monkeypatch):
    from pase_b200 import functional as Fn
    monkeypatch.setattr(Fn, "PRECISION", Fn.PRECISION)       # restored after the test
    Fn.set_precision(precision)
    gold, meta, model, batch = build_case(name)
    check_case(gold, meta, model, batch, "cpu")


def test_state_dict_keys_match_reference_layout():
    gold, meta, model, batch = build_case("pase_plus_workers_3200")
    keys = set(model.state_dict().keys())
    for k in gold:
        if k.startswith(("grad/", "gsample/")):
            assert k.split("/", 1)[1] in keys, k
    assert "regression_workers.0.blocks.0.deconv.weight" in keys
    assert "classification_workers.1.minion.W.bias" in keys


def test_fused_regression_heads_equal_unfused(emulated):
    """pase.fuse_regression_loss: same losses, same total, same gradients as the unfused heads
    (3xF16 GEMM mode; emulated kernels)."""
    from pase_b200 import functional as Fn
    assert Fn.PRECISION == "3xf16"
    res = {}
    for fused in (False, True):
        gold, meta, model, batch = build_case("pase_plus_workers_3200")
        model.fuse_regression_loss = fused
        random.seed(meta["seed"])
        h, chunk, preds, labels = model(batch, 1, "cpu")
        tot, losses = total_loss(model, preds, labels)
        tot.backward()
        res[fused] = (float(tot), {k: float(v) for k, v in losses.items()},
                      {k: p.grad.clone() for k, p in model.named_parameters()}, preds)
    (ta, la, ga, _), (tb, lb, gb, pb) = res[False], res[True]
    assert abs(ta - tb) <= 1e-5 * abs(ta)
    for k in la:
        assert abs(la[k] - lb[k]) <= 2e-5 * max(abs(la[k]), 1e-6), k
    for k in ga:
        if k.startswith("frontend.") and k.endswith(("conv.bias", "W.bias")):
            continue                      # analytically zero under train-mode BN: noise only
        scale = float(ga[k].abs().max())
        assert float((ga[k] - gb[k]).abs().max()) <= 2e-4 * scale + 1e-9, k
    # fused predictions are placeholders of the reference shape
    assert tuple(pb["lps"].shape) == tuple(res[False][3]["lps"].shape)
    assert pb["lps"].stride() == (0, 0, 0)
