"""Boundary proof against what the unmodified reference produced (tests/golden/boundary.pt,
written by tests/golden/make_golden.py::boundary_case from the reference's own code).

  (1) Training step: the reference's ``backprop_scheduler`` in 'base' mode
      (pase/models/WorkerScheduler/worker_scheduler.py:43-75), called as trainer.py:229-244
      calls it with one torch optimizer per worker + one for the frontend (trainer.py:86-143),
      drove the reference model for two optimisation steps.  The same step sequence drives the
      native ``pase_b200.pase.pase`` model on the same weights and batch; losses are compared
      step by step, then the weights after the second update.  (CUDA kernels replaced by their
      torch specs, tests/emul/; the GPU tests cover the kernels.)
  (2) Checkpoints: files written by the reference ``Saver`` / ``Model.save`` load into the
      native modules (``load_pretrained``, ``Model.load``); the native Saver writes the same
      index file, the same rotation and checkpoints of the same structure and content
      (pase/models/modules.py:151-373).
"""
import copy
import json
import os
import random

import pytest
import torch

import emul
from helpers import GOLDEN, load_golden, resolve_cfg, fill_state_dict, seeded_randn, sample_view
import pase_b200.ops as ops
from pase_b200 import encoder as enc, wf_builder
from pase_b200.frontend import WaveFe
from pase_b200.pase import pase as native_pase
from pase_b200.utils import parse_workers
from pase_b200 import modules as NM

# frontend of the checkpoint fixtures (tests/golden/make_golden.py::SAVER_CFG)
SAVER_CFG = {"kwidths": [31, 5, 3, 3, 3, 3, 3, 3], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [8, 8, 8, 8, 8, 8, 8, 8], "emb_dim": 8, "norm_out": True}


def _boundary():
    return torch.load(os.path.join(GOLDEN, "boundary.pt"), map_location="cpu")


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


def _optimizers(model, fe_lr=5e-4, min_lr=4e-4):
    """trainer.py:86-143: Adam per worker + Adam for the frontend."""
    fe = torch.optim.Adam(model.frontend.parameters(), lr=fe_lr)
    cls = {w.name: torch.optim.Adam(w.parameters(), lr=min_lr)
           for w in model.classification_workers}
    regr = {w.name: torch.optim.Adam(w.parameters(), lr=min_lr)
            for w in model.regression_workers}
    return fe, cls, regr


def _base_step(model, preds, labels, cls_opt, regr_opt, fe_opt):
    """One 'base' scheduler step: zero every optimizer, backward the weighted loss sum, step
    the worker optimizers, then the frontend's."""
    fe_opt.zero_grad()
    tot, losses = 0, {}
    for workers, opts in ((model.classification_workers, cls_opt),
                          (model.regression_workers, regr_opt), (model.regularizer_workers, None)):
        for w in workers:
            if opts is not None:
                opts[w.name].zero_grad()
            loss = w.loss_weight * w.loss(preds[w.name], labels[w.name])
            losses[w.name] = loss
            tot = tot + loss
    tot.backward()
    for opt in list(cls_opt.values()) + list(regr_opt.values()):
        opt.step()
    fe_opt.step()
    losses["total"] = tot
    return losses


def test_reference_scheduler_drives_native_model(emulated):
    gold = _boundary()
    _, meta = load_golden("pase_mini_workers_1600")
    fe_cfg, wcfg = resolve_cfg(meta["fe_cfg"]), meta["workers"]
    B, T, Tq, seed = meta["B"], meta["T"], meta["Tq"], meta["seed"]
    batch = {k: seeded_randn((B, 1, T), seed + 10 + i, 0.5)
             for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
    for i, w in enumerate(wcfg["regr"]):
        if w["name"] != "cchunk":
            batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)

    nat = native_pase(frontend_cfg=fe_cfg, minions_cfg=parse_workers(copy.deepcopy(wcfg))).train()
    nat.load_state_dict(fill_state_dict(nat.state_dict(), seed))
    fe_opt, cls_opt, regr_opt = _optimizers(nat)
    trace = []
    for it in range(2):
        random.seed(seed + it)                               # SPC-style host RNG, if any
        # trainer.py:229: h, chunk, preds, labels = self.model.forward(batch, alpha, device)
        h, chunk, preds, labels = nat.forward(dict(batch), 1, "cpu")
        losses = _base_step(nat, preds, labels, cls_opt, regr_opt, fe_opt)
        trace.append({k: float(v.detach()) for k, v in losses.items()})
    for it in range(2):
        ref = {k.split("/", 2)[2]: float(v) for k, v in gold.items()
               if k.startswith("sched/loss%d/" % it)}
        n = trace[it]
        assert set(ref) == set(n)
        for k in ref:
            # step 0: same weights -> fp32 parity; step 1: after one Adam update of every
            # parameter through each implementation's own gradients
            tol = 2e-4 if it == 0 else 2e-3
            assert abs(ref[k] - n[k]) <= tol * max(abs(ref[k]), 1e-3), (it, k, ref[k], n[k])
    # the update really happened (losses moved) and stayed in lock-step
    assert abs(float(gold["sched/loss1/total"]) - float(gold["sched/loss0/total"])) > 1e-4
    nsd = nat.state_dict()
    ref_keys = [k[len("sched/state/"):] if k.startswith("sched/state/") else k[len("sched/ssample/"):]
                for k in gold if k.startswith(("sched/state/", "sched/ssample/"))]
    assert sorted(ref_keys) == sorted(nsd.keys())
    for k, b in nsd.items():
        if not b.is_floating_point():
            continue
        a = gold.get("sched/state/" + k)
        if a is None:
            a, b = gold["sched/ssample/" + k], sample_view(b)
            gn = float(gold["sched/snorm/" + k])
            assert abs(float(nsd[k].double().norm()) - gn) <= 2e-3 * gn, k
        if k.startswith("frontend.") and (k.endswith("conv.bias") or k.endswith("W.bias")):
            # biases followed by train-mode BatchNorm: the gradient is analytically zero, both
            # implementations feed Adam rounding noise, and Adam turns ANY gradient into a
            # +-lr step -> the two may differ by up to 2 * lr per step, no more
            assert float((a - b).abs().max()) <= 2 * 5e-4 * 2 + 1e-6, k
            continue
        assert float((a - b).abs().max()) <= 2e-3 * max(float(a.abs().max()), 1e-3), k


def _dump(d, files):
    """writes the golden files {name: uint8 tensor} into directory d; -> d"""
    d = str(d)
    os.makedirs(d, exist_ok=True)
    for name, data in files.items():
        with open(os.path.join(d, name), "wb") as f:
            f.write(bytes(data.tolist()))
    return d


def test_saver_checkpoints_are_interchangeable(tmp_path):
    gold = _boundary()
    ref_files = {k[len("saver/file/"):]: v for k, v in gold.items() if k.startswith("saver/file/")}
    ref_index = json.loads(bytes(ref_files["PASE-checkpoints"].tolist()).decode())
    ref_ckpt = torch.load(os.path.join(_dump(tmp_path / "ref_written", ref_files),
                                       "weights_" + ref_index["current"]), map_location="cpu")
    ref_sd = ref_ckpt["state_dict"]
    nat_fe = wf_builder(dict(SAVER_CFG))
    assert list(ref_sd.keys()) == list(nat_fe.state_dict().keys())
    nat_opt = torch.optim.Adam(nat_fe.parameters(), lr=1e-3)

    # --- reference writes, native reads (Saver directory + bare ckpt file) -------------
    d1 = str(tmp_path / "ref_written")
    ns = NM.Saver(nat_fe, d1, max_ckpts=2, optimizer=nat_opt, prefix="PASE-")
    assert ns.read_latest_checkpoint() == ref_index["current"]
    assert ns.load_weights() is True
    for k, v in ref_sd.items():
        assert torch.equal(v, nat_fe.state_dict()[k]), k
    assert ns.load_ckpt_step(ns.read_latest_checkpoint()) == 40
    # README.md:28-33 usage: load_pretrained(path, load_last=True)
    nat2 = wf_builder(dict(SAVER_CFG))
    ckpt = os.path.join(d1, "weights_" + ref_index["current"])
    nat2.load_pretrained(ckpt, load_last=True, verbose=False)
    for k, v in ref_sd.items():
        assert torch.equal(v, nat2.state_dict()[k]), k
    # load_last=False drops the last two keys -> the reference raises on a key-count mismatch
    with pytest.raises(ValueError, match="LOADING DIFFERENT NUM OF KEYS"):
        wf_builder(dict(SAVER_CFG)).load_pretrained(ckpt, load_last=False, verbose=False)

    # --- native writes the same sequence: identical index file, rotation and contents -----
    d2 = str(tmp_path / "nat_written")
    ns2 = NM.Saver(nat_fe, d2, max_ckpts=2, optimizer=nat_opt, prefix="PASE-")
    for step in (10, 20, 30, 40):
        ns2.save("FE_e%d" % (step // 10), step)
    assert json.load(open(os.path.join(d2, "PASE-checkpoints"))) == ref_index
    assert sorted(os.listdir(d2)) == json.loads(gold["saver/listing"])
    # what the reference reads back from a native checkpoint is what it wrote itself
    nat_ckpt = torch.load(os.path.join(d2, "weights_" + ref_index["current"]), map_location="cpu")
    assert list(nat_ckpt.keys()) == list(ref_ckpt.keys()) and nat_ckpt["step"] == ref_ckpt["step"]
    assert list(nat_ckpt["state_dict"].keys()) == list(ref_sd.keys())
    for k, v in ref_sd.items():
        assert torch.equal(v, nat_ckpt["state_dict"][k]), k
    assert nat_ckpt["optimizer"]["param_groups"] == ref_ckpt["optimizer"]["param_groups"]

    # Model.save / Model.load (modules.py:311-340) through the model's own saver
    model_files = {k[len("saver/model_file/"):]: v for k, v in gold.items()
                   if k.startswith("saver/model_file/")}
    d3 = _dump(tmp_path / "model_api", model_files)
    nat3 = wf_builder(dict(SAVER_CFG))
    nat3.name = gold["saver/model_name"]
    nat3.load(d3)
    for k, v in ref_sd.items():
        assert torch.equal(v, nat3.state_dict()[k]), k
    pasep = wf_builder(resolve_cfg("cfg/frontend/PASE+.cfg"))
    assert pasep.get_total_params() == gold["saver/pasep_total_params"] == 7832896
