"""Drop-in for ``pase.models.pase.pase`` (pase.py:241-356): the encoder plus the
fan-out of self-supervised workers, same constructor, same
``forward(x, alpha=1, device=None) -> (h, chunk, preds, labels)`` protocol, same
``frontend`` / ``regression_workers`` / ``classification_workers`` attributes and
state_dict keys, so the reference trainer (trainer.py:229, worker_scheduler.py:43-75)
drives it unchanged.  Heads consume the encoder's channel-last output directly.
"""
import torch
import torch.nn as nn

from .modules import Model
from .frontend import wf_builder
from .minions import minion_maker, cls_worker_maker, RowsInput


class pase(Model):
    def __init__(self, frontend=None, frontend_cfg=None, minions_cfg=None,
                 cls_lst=["mi", "cmi", "spc"], regr_lst=["chunk", "lps", "mfcc", "prosody"],
                 pretrained_ckpt=None, name="adversarial"):
        super().__init__(name=name)
        if minions_cfg is None or len(minions_cfg) < 1:
            raise ValueError('Please specify a stack of minions config with at least 1 minion.')
        self.frontend = frontend if frontend is not None else wf_builder(frontend_cfg)
        self.cls_lst, self.reg_lst = cls_lst, regr_lst
        ninp = self.frontend.emb_dim
        self.regression_workers = nn.ModuleList()
        self.classification_workers = nn.ModuleList()
        self.regularizer_workers = []
        self.fwd_cchunk = False
        # opt-in: fuse each MLP regression head's output layer with its contextualised MSE
        # (the (B, F*r, T) prediction -- 551 MB for the lps heads at B=32 -- is never
        # stored; preds[name] is then a placeholder carrying the reduced loss).  Off by default:
        # the trainer's histogram logging (trainer.py:405-413) reads preds[name].
        self.fuse_regression_loss = False
        for kind, cfg_lst in minions_cfg.items():
            for cfg in cfg_lst:
                cfg = dict(cfg)
                cfg['num_inputs'] = ninp
                if kind == 'cls':
                    self.classification_workers.append(cls_worker_maker(cfg, ninp))
                elif kind == 'regr':
                    self.regression_workers.append(minion_maker(cfg))
                elif kind == 'regu':
                    raise NotImplementedError("regularizer workers are not part of "
                                              "workers.cfg / workers+.cfg")
        if pretrained_ckpt is not None:
            self.load_pretrained(pretrained_ckpt, load_last=True)

    def forward(self, x, alpha=1, device=None):
        if device is None:
            device = self.frontend.W.weight.device
        x_ = dict(x)
        if not self.fwd_cchunk:
            x_.pop('cchunk', None)               # pase.py:314-317
        h = self.frontend(x_, device)
        rows = self.frontend.last_output_ntc     # (k*B*T', emb) channel-last, same autograd node
        h, chunk = h                             # (embedding tuple or tensor, chunk)
        nchunks = len(h) if isinstance(h, tuple) else 1
        B, Tq = chunk.shape[0], chunk.shape[2]
        per = B * Tq
        tagged = []
        for i in range(nchunks):
            t = h[i] if isinstance(h, tuple) else h
            t._pase_rows_in = RowsInput(rows[i * per:(i + 1) * per], B, Tq)
            tagged.append(t)
        chunk._pase_rows_in = tagged[0]._pase_rows_in

        preds, labels = {}, {}
        for worker in self.regression_workers:
            lab = x[worker.name].to(device).detach()
            if self.fuse_regression_loss and hasattr(worker, "_can_fuse"):
                y = worker(chunk, alpha, label=lab)
            else:
                y = worker(chunk, alpha)
            preds[worker.name] = y
            labels[worker.name] = lab
        for worker in self.classification_workers:
            if worker.name in ("spc", "gap"):
                y, label = worker(chunk, alpha, device=device)
            else:
                y, label = worker(h, alpha, device=device)
            preds[worker.name] = y
            labels[worker.name] = label
        return h, chunk, preds, labels


def total_loss(model, preds, labels):
    """sum_w loss_weight_w * loss_w(pred, label): the 'base' backprop scheduler
    (worker_scheduler.py:43-62)."""
    tot, losses = 0., {}
    for w in list(model.classification_workers) + list(model.regression_workers):
        l = w.loss_weight * w.loss(preds[w.name], labels[w.name])
        losses[w.name] = l
        tot = tot + l
    return tot, losses


def eval_losses(model, preds, labels):
    """The losses of a validation batch as the reference trainer's ``_eval`` computes them
    (trainer.py:303-326): each worker's UNWEIGHTED loss, classification workers first, then
    regression workers, and their fp32 sum in that order."""
    tot, losses = 0., {}
    for w in list(model.classification_workers) + list(model.regression_workers):
        l = w.loss(preds[w.name], labels[w.name])
        losses[w.name] = l
        tot = tot + l
    return tot, losses
