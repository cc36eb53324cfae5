"""Reference harness -- TEST INFRASTRUCTURE, container-only.

Imports the UNMODIFIED reference (a read-only checkout of santi-pdp/pase at
$PASE_REFERENCE_ROOT) on CPU so that (a) the CPU restatement in
``oracle/pase_oracle.py`` can be pinned against the real thing and (b) golden
vectors can be generated (``tests/golden/make_golden.py``).  The tests and the
benchmark never import this module: they run without the reference; it raises
ImportError when the reference tree is absent.

Shims (SURVEY.md section 8c):
  * ``soundfile``  -- import-only dependency of pase/models/pase.py:15.
  * ``torchqrnn``  -- un-vendored, un-pinned third-party dependency
    (requirements.txt:16).  The stand-in below restates the published
    algorithm of salesforce/pytorch-qrnn (QRNNLayer.forward + CPUForgetMult)
    as called at pase/models/modules.py:52 (window=2, one layer per entry in
    ``layers``).  Parity for the QRNN is therefore "unpinned" against
    torchqrnn itself (see DESIGN.md).
"""
import os
import sys
import types
import json
import contextlib
import io

REF_ROOT = os.environ.get("PASE_REFERENCE_ROOT", "")


def reference_available():
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "pase", "models"))


def _install_shims():
    import torch
    import torch.nn as nn

    if "soundfile" not in sys.modules:
        sys.modules["soundfile"] = types.ModuleType("soundfile")

    if "torchqrnn" not in sys.modules:
        class _QRNNLayer(nn.Module):
            def __init__(self, input_size, hidden_size, window):
                super().__init__()
                self.window = window
                self.hidden_size = hidden_size
                self.linear = nn.Linear(window * input_size, 3 * hidden_size)

            def forward(self, X, hidden=None):
                # X: (T, N, C).  window=2: source is [x_t, x_{t-1}] with x_{-1}=0
                Xm1 = torch.cat([torch.zeros_like(X[:1]), X[:-1]], 0)
                Y = self.linear(torch.cat([X, Xm1], 2))
                Z, F, O = Y.chunk(3, dim=2)
                Z = torch.tanh(Z)
                F = torch.sigmoid(F)
                cs = []
                c = hidden
                for t in range(X.shape[0]):
                    c = F[t] * Z[t] if c is None else F[t] * Z[t] + (1 - F[t]) * c
                    cs.append(c)
                C = torch.stack(cs, 0)
                H = torch.sigmoid(O) * C
                return H, C[-1:]

        class QRNN(nn.Module):
            def __init__(self, input_size, hidden_size, num_layers=1,
                         dropout=0, window=1, use_cuda=True, **kw):
                super().__init__()
                self.layers = nn.ModuleList(
                    [_QRNNLayer(input_size if l == 0 else hidden_size,
                                hidden_size, window)
                     for l in range(num_layers)])

            def forward(self, X, hidden=None):
                nh = []
                for layer in self.layers:
                    X, h = layer(X, None)
                    nh.append(h)
                return X, torch.cat(nh, 0)

        mod = types.ModuleType("torchqrnn")
        mod.QRNN = QRNN
        sys.modules["torchqrnn"] = mod


def import_reference():
    """Returns the reference's ``pase`` package (imported from REF_ROOT)."""
    if not reference_available():
        raise ImportError("reference tree not present at %s" % REF_ROOT)
    sys.dont_write_bytecode = True
    _install_shims()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import pase  # noqa: F401
    import pase.models.frontend  # noqa: F401
    return sys.modules["pase"]


def ref_cfg_path(rel):
    return os.path.join(REF_ROOT, rel)


def build_ref_frontend(cfg):
    """cfg: dict or path relative to the reference root."""
    import_reference()
    from pase.models.frontend import wf_builder
    if isinstance(cfg, str):
        cfg = ref_cfg_path(cfg)
    with contextlib.redirect_stdout(io.StringIO()):
        return wf_builder(cfg)


def load_worker_cfg(rel_or_dict):
    """workers cfg -> dict with ContextualizedLoss objects, 'transform' popped
    (train.py:64 does the pop in the real flow)."""
    import_reference()
    from pase.utils import worker_parser
    if isinstance(rel_or_dict, dict):
        import tempfile
        with tempfile.NamedTemporaryFile("w", suffix=".cfg", delete=False) as f:
            json.dump(rel_or_dict, f)
            path = f.name
    else:
        path = ref_cfg_path(rel_or_dict)
    with contextlib.redirect_stdout(io.StringIO()):
        mcfg = worker_parser(path)
    for ws in mcfg.values():
        for w in ws:
            w.pop("transform", None)
    return mcfg


def build_ref_pase(frontend_cfg, workers_cfg):
    import_reference()
    from pase.models.pase import pase as ref_pase
    if isinstance(frontend_cfg, str):
        with open(ref_cfg_path(frontend_cfg)) as f:
            frontend_cfg = json.load(f)
    mcfg = load_worker_cfg(workers_cfg)
    cls_lst = [w["name"] for w in mcfg.get("cls", [])]
    regr_lst = [w["name"] for w in mcfg.get("regr", [])]
    with contextlib.redirect_stdout(io.StringIO()):
        model = ref_pase(frontend_cfg=frontend_cfg, minions_cfg=mcfg,
                         cls_lst=cls_lst, regr_lst=regr_lst)
    return model


def ref_total_loss(model, preds, labels):
    """worker_scheduler.py:43-62 ('base' mode): sum_w loss_weight * loss."""
    tot = 0
    losses = {}
    for w in list(model.classification_workers) + list(model.regression_workers):
        l = w.loss_weight * w.loss(preds[w.name], labels[w.name])
        losses[w.name] = l
        tot = tot + l
    return tot, losses
