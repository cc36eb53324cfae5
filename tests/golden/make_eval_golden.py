"""Generates tests/golden/eval.pt from the UNMODIFIED reference's validation pass (needs a checkout
of santi-pdp/pase).  Run:  PASE_REFERENCE_ROOT=<checkout> python tests/golden/make_eval_golden.py

The reference trainer's ``_eval`` (trainer.py:282-337), called with a stub ``self``, on the
pase_mini_workers_1600 model of make_golden.py with an SPC head and without the cchunk decoder,
after two 'base' training steps (so the BatchNorm running statistics have moved).  Stored: the
model state the pass ran on and its running_loss (every worker's unweighted loss and 'total',
per batch) over EVAL_BATCHES seeded batches, the host RNG seeded before the pass.  The decoder is
left out to keep the fixture small (its weights are half of the state); it has no BatchNorm, so
eval mode does not change it, and pase_mini_workers_1600 covers its forward.
"""
import contextlib
import copy
import io
import json
import os
import random
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)
import ref_harness as rh                      # noqa: E402
from detweights import fill_state_dict, seeded_randn  # noqa: E402
from make_golden import MINI_CFG, MINI_WORKERS  # noqa: E402

# MINI_WORKERS without the decoder, plus an SPC head whose frame ranges fit the T' = 10 frames of
# a 1600-sample chunk (seq_pad + ctxt_frames = 3: t in [4, 7))
EVAL_WORKERS = {
    "regr": [w for w in MINI_WORKERS["regr"] if w["name"] != "cchunk"],
    "cls": MINI_WORKERS["cls"] + [
        {"num_outputs": 1, "dropout": 0, "hidden_size": 64, "hidden_layers": 1, "name": "spc",
         "type": "spc", "ctxt_frames": 2, "seq_pad": 1, "skip": False,
         "loss": "BCEWithLogitsLoss"}],
}
EVAL_BATCHES = 3


def eval_batch(B, T, Tq, wcfg, seed):
    """A seeded batch: the four waveforms and one label per regression worker (the test
    regenerates the validation batches with the same function)."""
    batch = {k: seeded_randn((B, 1, T), seed + i, 0.5)
             for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
    for i, w in enumerate(wcfg["regr"]):
        if w["name"] != "cchunk":
            batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)
    return batch


def eval_case():
    rh.import_reference()
    from pase.models.WorkerScheduler.worker_scheduler import backprop_scheduler
    from pase.models.WorkerScheduler.trainer import trainer as RefTrainer
    seed, B, T = 8, 2, 1600
    wcfg = json.loads(json.dumps(EVAL_WORKERS))
    model = rh.build_ref_pase(dict(MINI_CFG), copy.deepcopy(wcfg)).train()
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    with torch.no_grad():
        model.eval()
        Tq = model.frontend(seeded_randn((B, 1, T), 0, 0.5)).shape[2]
        model.train()
    train_batch = eval_batch(B, T, Tq, wcfg, seed + 10)
    sched = backprop_scheduler(model, mode="base")
    fe_opt = torch.optim.Adam(model.frontend.parameters(), lr=5e-4)
    cls_opt = {w.name: torch.optim.Adam(w.parameters(), lr=4e-4)
               for w in model.classification_workers}
    regr_opt = {w.name: torch.optim.Adam(w.parameters(), lr=4e-4)
                for w in model.regression_workers}
    for it in range(2):
        random.seed(seed + it)
        _, _, preds, labels = model.forward(dict(train_batch), 1, "cpu")
        sched(preds, labels, cls_opt, regr_opt, fe_opt, device="cpu")
    out = {"meta": json.dumps({"fe_cfg": MINI_CFG, "workers": wcfg, "B": B, "T": T, "Tq": Tq,
                               "seed": seed, "batches": EVAL_BATCHES})}
    for k, v in model.state_dict().items():
        out["state/" + k] = v.detach().clone()
    # batch i: eval_batch(B, T, Tq, workers, seed + 1000 + 200 * i)
    batches = [eval_batch(B, T, Tq, wcfg, seed + 1000 + 200 * i) for i in range(EVAL_BATCHES)]
    logged = {}
    stub = types.SimpleNamespace(model=model, va_bpe=EVAL_BATCHES, log_freq=10 ** 9, bpe=10 ** 9,
                                 eval_logger=lambda rl, epoch, pbar: logged.update(rl))
    random.seed(seed + 50)
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        RefTrainer._eval(stub, [dict(b) for b in batches], epoch=0, device="cpu")
    out["names"] = json.dumps(list(logged))
    for k, v in logged.items():
        assert len(v) == EVAL_BATCHES, (k, v)
        out["loss/" + k] = torch.tensor(v, dtype=torch.float64)
    torch.save(out, os.path.join(HERE, "eval.pt"))
    print("eval", os.path.getsize(os.path.join(HERE, "eval.pt")),
          {k: [round(x, 5) for x in v] for k, v in logged.items()})


if __name__ == "__main__":
    torch.set_num_threads(8)
    eval_case()
