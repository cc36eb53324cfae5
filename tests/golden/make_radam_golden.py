"""Generates tests/golden/radam.pt from the UNMODIFIED reference RAdam
(pase/models/WorkerScheduler/radam.py) and Saver (pase/models/modules.py).  Run:
    PASE_REFERENCE_ROOT=<checkout> python tests/golden/make_radam_golden.py

One reference ``RAdam`` instance per "module", each with one parameter group, the layout the
reference trainer builds for ``--fe_opt radam`` / ``--min_opt radam`` (trainer.py:86-135).
The parameters have odd sizes; the instances differ in lr, weight decay and betas.  Seeded
gradients drive STEPS steps, so every instance crosses rho = 5 (step 6 for beta2 = 0.999,
also step 6 for 0.99); after step LR_CHANGE_AFTER every lr is multiplied by LR_FACTOR, as an
LR scheduler would.

Contents:
  meta                    dict(steps, lr_change_after, lr_factor, saver_instance, saver_steps)
  cfg/<i>                 dict(lr, betas, weight_decay, shapes)
  init/<i>/<j>            parameter j of instance i before the first step
  grad/<i>/<s>/<j>        its gradient at step s (1-based)
  param/<i>/<s>/<j>       its value after step s
  state8/<i>              the instance's state_dict() after step 8
  saver/file/<name>       the files the reference Saver writes for instance SAVER_INSTANCE (a
                          module holding its parameters) after steps 4 and 8, prefix
                          'M-radam-', as uint8 tensors
"""
import contextlib
import copy
import io
import os
import shutil
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness as rh                      # noqa: E402

STEPS = 12
LR_CHANGE_AFTER = 7
LR_FACTOR = 0.5
SAVER_INSTANCE = 1
SAVER_STEPS = (4, 8)
INSTANCES = [
    dict(lr=2e-3, betas=(0.9, 0.999), weight_decay=0.0, shapes=[(7, 13), (13,)]),
    dict(lr=1e-2, betas=(0.9, 0.999), weight_decay=1e-2, shapes=[(5, 3, 3), (5,), (1,)]),
    dict(lr=5e-3, betas=(0.8, 0.99), weight_decay=0.0, shapes=[(29,), (3, 11)]),
    dict(lr=3e-4, betas=(0.8, 0.99), weight_decay=1e-2, shapes=[(17,), (2, 9)]),
]


class _Holder(torch.nn.Module):
    """What a reference Saver wraps: a module whose state_dict holds the parameters."""

    def __init__(self, params):
        super().__init__()
        for j, p in enumerate(params):
            self.register_parameter("p%d" % j, p)


def _file_bytes(path):
    with open(path, "rb") as f:
        return torch.tensor(list(f.read()), dtype=torch.uint8)


def main():
    rh.import_reference()
    from pase.models.WorkerScheduler.radam import RAdam
    from pase.models.modules import Saver as RefSaver
    out = {"meta": dict(steps=STEPS, lr_change_after=LR_CHANGE_AFTER, lr_factor=LR_FACTOR,
                        saver_instance=SAVER_INSTANCE, saver_steps=SAVER_STEPS)}
    gen = torch.Generator().manual_seed(2026)
    params, opts = [], []
    for i, c in enumerate(INSTANCES):
        out["cfg/%d" % i] = dict(c)
        ps = [torch.nn.Parameter(torch.randn(s, generator=gen)) for s in c["shapes"]]
        for j, p in enumerate(ps):
            out["init/%d/%d" % (i, j)] = p.detach().clone()
        params.append(ps)
        opts.append(RAdam(ps, lr=c["lr"], betas=c["betas"], weight_decay=c["weight_decay"]))
    saver_dir = tempfile.mkdtemp()
    holder = _Holder(params[SAVER_INSTANCE])
    saver = RefSaver(holder, saver_dir, optimizer=opts[SAVER_INSTANCE], prefix="M-radam-")
    with contextlib.redirect_stdout(io.StringIO()):
        for s in range(1, STEPS + 1):
            if s == LR_CHANGE_AFTER + 1:
                for o in opts:
                    for g in o.param_groups:
                        g["lr"] *= LR_FACTOR
            for i, (ps, o) in enumerate(zip(params, opts)):
                # gradients of a spread of scales, so eps matters for some elements
                for j, p in enumerate(ps):
                    g = torch.randn(p.shape, generator=gen) * 10.0 ** (j - 2)
                    out["grad/%d/%d/%d" % (i, s, j)] = g.clone()
                    p.grad = g
                o.step()
                for j, p in enumerate(ps):
                    out["param/%d/%d/%d" % (i, s, j)] = p.detach().clone()
                if s == 8:
                    out["state8/%d" % i] = copy.deepcopy(o.state_dict())
            if s in SAVER_STEPS:
                saver.save("W", s)
    for name in sorted(os.listdir(saver_dir)):
        out["saver/file/" + name] = _file_bytes(os.path.join(saver_dir, name))
    shutil.rmtree(saver_dir)
    path = os.path.join(HERE, "radam.pt")
    torch.save(out, path)
    print("radam", os.path.getsize(path), sorted(k for k in out if k.startswith("saver/")))


if __name__ == "__main__":
    main()
