"""Generates tests/golden/*.pt from the UNMODIFIED reference (needs a checkout of
santi-pdp/pase).  Run:  PASE_REFERENCE_ROOT=<checkout> python tests/golden/make_golden.py

Every case: deterministic parameters (detweights.fill_state_dict) are loaded
into the reference module, seeded inputs are pushed through the reference's own
forward / autograd on CPU, and outputs + gradients are stored.  Gradients of
tensors with more than FULL_MAX elements are stored as a strided sample plus
their L2 norm.
"""
import os
import sys
import json
import random
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)
import ref_harness as rh                      # noqa: E402
from detweights import fill_state_dict, seeded_randn, sample_view  # noqa: E402

FULL_MAX = 20000

MINI_CFG = {
    "kwidths": [63, 10, 5, 4, 5, 5, 5, 5],
    "strides": [1, 10, 2, 1, 2, 1, 2, 2],
    "fmaps": [16, 16, 32, 32, 32, 48, 48, 64],
    "emb_dim": 40, "rnn_dim": 64,
    "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1,
}
MINI_NORNN_CFG = {
    "kwidths": [31, 20, 11, 11, 11, 11, 11, 11],
    "strides": [1, 10, 2, 1, 2, 1, 2, 2],
    "fmaps": [8, 8, 16, 16, 24, 24, 32, 32],
    "emb_dim": 20, "norm_out": True,
}
# checkpoint-format fixtures only (small files)
SAVER_CFG = {
    "kwidths": [31, 5, 3, 3, 3, 3, 3, 3],
    "strides": [1, 10, 2, 1, 2, 1, 2, 2],
    "fmaps": [8, 8, 8, 8, 8, 8, 8, 8],
    "emb_dim": 8, "norm_out": True,
}
MINI_WORKERS = {
    "regr": [
        {"num_outputs": 1, "dropout": 0, "dropout_time": 0.0, "hidden_layers": 1,
         "name": "cchunk", "type": "decoder", "hidden_size": 16,
         "fmaps": [48, 32, 24], "strides": [4, 4, 10], "kwidths": [30, 30, 30],
         "loss": "L1Loss"},
        {"num_outputs": 33, "dropout": 0, "hidden_size": 64, "hidden_layers": 1,
         "name": "lps", "context": 1, "r": 7, "loss": "MSELoss", "skip": False},
        {"num_outputs": 12, "dropout": 0, "hidden_size": 64, "hidden_layers": 1,
         "name": "prosody", "context": 1, "r": 3, "loss": "MSELoss", "skip": False},
        {"num_outputs": 20, "dropout": 0, "hidden_size": 64, "hidden_layers": 1,
         "name": "mfcc", "loss": "MSELoss", "skip": False},
    ],
    "cls": [
        {"num_outputs": 1, "dropout": 0, "hidden_size": 64, "hidden_layers": 1,
         "name": "mi", "loss": "BCEWithLogitsLoss", "skip": False,
         "keys": ["chunk", "chunk_ctxt", "chunk_rand"]},
        {"num_outputs": 1, "dropout": 0, "hidden_size": 64, "hidden_layers": 1,
         "name": "cmi", "augment": True, "loss": "BCEWithLogitsLoss", "skip": False,
         "keys": ["chunk", "chunk_ctxt", "chunk_rand"]},
    ],
}


def _store_grad(out, key, g):
    if g.numel() <= FULL_MAX:
        out["grad/" + key] = g.detach().clone()
    else:
        out["gsample/" + key] = sample_view(g.detach())
        out["gnorm/" + key] = g.detach().double().norm().float()


def encoder_case(name, cfg, N, T, training, seed, with_grads=True):
    m = rh.build_ref_frontend(dict(cfg) if isinstance(cfg, dict) else cfg)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed))
    m.train(training)
    x = seeded_randn((N, 1, T), seed + 1, 0.5)
    out = {"meta": json.dumps({"cfg": cfg, "N": N, "T": T, "training": training,
                               "seed": seed})}
    if training and with_grads:
        y = m(x)
        cot = seeded_randn(tuple(y.shape), seed + 2)
        (y * cot).sum().backward()
        for k, p in m.named_parameters():
            _store_grad(out, k, p.grad)
        for k, b in m.named_buffers():
            out["stat/" + k] = b.detach().clone()
    else:
        with torch.no_grad():
            y = m(x)
    out["y"] = y.detach().clone()
    # per-block frame counts, straight from the reference blocks
    lens, h = [], x
    with torch.no_grad():
        m.eval()
        for blk in m.blocks:
            h = blk(h)
            lens.append(h.shape[2])
    out["frame_counts"] = torch.tensor(lens)
    torch.save(out, os.path.join(HERE, name + ".pt"))
    print(name, tuple(y.shape), lens)


def _file_bytes(path):
    with open(path, "rb") as f:
        return torch.tensor(list(f.read()), dtype=torch.uint8)


def boundary_case():
    """boundary.pt: what the reference's own training-step code and checkpoint code produce,
    for tests/test_reference_boundary.py.
      sched/*: backprop_scheduler('base') with one Adam per worker + one for the frontend
               (trainer.py:86-143, 229-244) driving the reference pase model of
               pase_mini_workers_1600 for two steps: per-step losses and the final weights
               (tensors above FULL_MAX elements as a strided sample plus their L2 norm).
      saver/*: files the reference Saver writes for a SAVER_CFG frontend (four saves,
               max_ckpts=2, prefix 'PASE-'), and those of Model.save(dir, 5)."""
    import copy
    import tempfile
    rh.import_reference()
    from pase.models.WorkerScheduler.worker_scheduler import backprop_scheduler
    from pase.models.modules import Saver as RefSaver
    out = {}
    seed, B, T = 8, 2, 1600
    wcfg = json.loads(json.dumps(MINI_WORKERS))
    model = rh.build_ref_pase(dict(MINI_CFG), copy.deepcopy(wcfg)).train()
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    batch = {k: seeded_randn((B, 1, T), seed + 10 + i, 0.5)
             for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
    with torch.no_grad():
        model.eval()
        Tq = model.frontend(batch["chunk"]).shape[2]
        model.train()
    for i, w in enumerate(wcfg["regr"]):
        if w["name"] != "cchunk":
            batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)
    sched = backprop_scheduler(model, mode="base")
    fe_opt = torch.optim.Adam(model.frontend.parameters(), lr=5e-4)
    cls_opt = {w.name: torch.optim.Adam(w.parameters(), lr=4e-4)
               for w in model.classification_workers}
    regr_opt = {w.name: torch.optim.Adam(w.parameters(), lr=4e-4)
                for w in model.regression_workers}
    for it in range(2):
        random.seed(seed + it)
        h, chunk, preds, labels = model.forward(dict(batch), 1, "cpu")
        losses, _ = sched(preds, labels, cls_opt, regr_opt, fe_opt, device="cpu")
        for k, v in losses.items():
            out["sched/loss%d/%s" % (it, k)] = torch.tensor(float(v.detach()), dtype=torch.float64)
    for k, v in model.state_dict().items():
        if v.numel() <= FULL_MAX:
            out["sched/state/" + k] = v.detach().clone()
        else:
            out["sched/ssample/" + k] = sample_view(v.detach())
            out["sched/snorm/" + k] = v.detach().double().norm()

    fe = rh.build_ref_frontend(dict(SAVER_CFG))
    fe.load_state_dict(fill_state_dict(fe.state_dict(), 7))
    opt = torch.optim.Adam(fe.parameters(), lr=1e-3)
    with tempfile.TemporaryDirectory() as d:
        d1 = os.path.join(d, "saver")
        rs = RefSaver(fe, d1, max_ckpts=2, optimizer=opt, prefix="PASE-")
        import contextlib
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            for step in (10, 20, 30, 40):
                rs.save("FE_e%d" % (step // 10), step)
            d3 = os.path.join(d, "model_api")
            fe.save(d3, 5)
        out["saver/listing"] = json.dumps(sorted(os.listdir(d1)))
        for name in sorted(os.listdir(d1)):
            out["saver/file/" + name] = _file_bytes(os.path.join(d1, name))
        out["saver/model_name"] = fe.name
        for name in sorted(os.listdir(d3)):
            out["saver/model_file/" + name] = _file_bytes(os.path.join(d3, name))
    out["saver/pasep_total_params"] = rh.build_ref_frontend("cfg/frontend/PASE+.cfg").get_total_params()
    torch.save(out, os.path.join(HERE, "boundary.pt"))
    print("boundary", os.path.getsize(os.path.join(HERE, "boundary.pt")))


def frame_count_table():
    m = rh.build_ref_frontend("cfg/frontend/PASE+.cfg").eval()
    table = {}
    for T in [1000, 12345, 15999, 16000, 16001, 31999, 32000, 48000]:
        h = torch.zeros(1, 1, T)
        lens = []
        with torch.no_grad():
            for blk in m.blocks:
                h = blk(h)
                lens.append(h.shape[2])
        table[T] = lens
    with open(os.path.join(HERE, "frame_counts.json"), "w") as f:
        json.dump(table, f, indent=1)
    print("frame_counts", table)


def small_kats():
    rh.import_reference()
    from pase.losses import ContextualizedLoss
    from pase.models.modules import SincConv_fast, select_output
    import torch.nn as nn
    out = {}
    lab = seeded_randn((2, 3, 9), 11)
    for r in (3, 7):
        out["ctx_r%d" % r] = ContextualizedLoss(nn.MSELoss(), r).contextualize_r(lab)
    out["ctx_label"] = lab
    sc = SincConv_fast(1, 64, 251, padding="SAME")
    with torch.no_grad():
        sc(torch.zeros(1, 1, 600))
    out["sinc_low"] = sc.low_hz_.detach().clone()
    out["sinc_band"] = sc.band_hz_.detach().clone()
    out["sinc_filters"] = sc.filters.detach().clone()
    h = seeded_randn((2, 5, 7), 12)
    for mode in ("avg_norm", "avg_concat", "avg_norm_concat"):
        out["sel_" + mode] = select_output(h, mode)
    out["sel_in"] = h
    torch.save(out, os.path.join(HERE, "kats.pt"))
    print("kats ok")


def pase_case(name, fe_cfg, workers, B, T, seed):
    model = rh.build_ref_pase(dict(fe_cfg) if isinstance(fe_cfg, dict) else fe_cfg,
                              json.loads(json.dumps(workers)) if isinstance(workers, dict) else workers)
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    model.train()
    Tq = None
    batch = {}
    for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"]):
        batch[k] = seeded_randn((B, 1, T), seed + 10 + i, 0.5)
    # labels: one per regression worker (cchunk already present)
    wcfg = workers if isinstance(workers, dict) else json.load(open(rh.ref_cfg_path(workers)))
    with torch.no_grad():
        model.eval()
        Tq = model.frontend(batch["chunk"]).shape[2]
        model.train()
    for i, w in enumerate(wcfg["regr"]):
        if w["name"] == "cchunk":
            continue
        batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)
    random.seed(seed)
    h, chunk, preds, labels = model(batch, 1, "cpu")
    tot, losses = rh.ref_total_loss(model, preds, labels)
    tot.backward()
    out = {"meta": json.dumps({"fe_cfg": fe_cfg, "workers": wcfg, "B": B, "T": T,
                               "seed": seed, "Tq": Tq})}
    out["total"] = tot.detach().clone()
    for k, v in losses.items():
        out["loss/" + k] = v.detach().clone()
    out["chunk"] = chunk.detach().clone()
    for k, v in preds.items():
        if v.numel() <= FULL_MAX:
            out["pred/" + k] = v.detach().clone()
        else:
            out["psample/" + k] = sample_view(v.detach())
    for k, p in model.named_parameters():
        _store_grad(out, k, p.grad)
    torch.save(out, os.path.join(HERE, name + ".pt"))
    print(name, float(tot), {k: round(float(v), 5) for k, v in losses.items()})


if __name__ == "__main__":
    torch.set_num_threads(8)
    frame_count_table()
    small_kats()
    # BASELINE.json config 0: PASE.cfg eval forward (1,1,16000) -> (1,100,100)
    encoder_case("enc_pase_eval_16000", "cfg/frontend/PASE.cfg", 1, 16000, False, 0)
    encoder_case("enc_pasep_eval_3200", "cfg/frontend/PASE+.cfg", 2, 3200, False, 1)
    encoder_case("enc_pasep_train_3200", "cfg/frontend/PASE+.cfg", 2, 3200, True, 2)
    encoder_case("enc_pasep_train_4001", "cfg/frontend/PASE+.cfg", 3, 4001, True, 3)
    encoder_case("enc_pase_train_2400", "cfg/frontend/PASE.cfg", 2, 2400, True, 4)
    encoder_case("enc_mini_train_2000", MINI_CFG, 3, 2000, True, 5)
    encoder_case("enc_mini_train_1763", MINI_CFG, 2, 1763, True, 6)
    encoder_case("enc_mininornn_train_1600", MINI_NORNN_CFG, 2, 1600, True, 7)
    pase_case("pase_mini_workers_1600", MINI_CFG, MINI_WORKERS, 2, 1600, 8)
    pase_case("pase_plus_workers_3200", "cfg/frontend/PASE+.cfg",
              "cfg/workers/workers+.cfg", 2, 3200, 9)
    boundary_case()
