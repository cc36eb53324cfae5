"""Worker heads + pase wrapper on the GPU (C-ABI kernels) against the reference goldens."""
import pytest
import torch

from test_heads_emulated import build_case, check_case
from helpers import assert_close, seeded_randn
from pase_b200.minions import MLPMinion
from pase_b200.losses import ContextualizedLoss
import pase_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["pase_mini_workers_1600", "pase_plus_workers_3200"])
def test_pase_workers_match_reference_golden(name):
    gold, meta, model, batch = build_case(name, "cuda")
    check_case(gold, meta, model, batch, "cuda", rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize("precision", ["fp32", "3xf16"])
def test_pase_workers_step_is_reproducible(precision):
    """Two identical forward + backward passes of the PASE+ encoder with its worker heads give
    the same loss and the same gradient bits (no sum in the step depends on scheduling)."""
    import random
    from pase_b200.pase import total_loss
    from pase_b200 import functional as Fn
    prev = Fn.PRECISION
    Fn.set_precision(precision)
    try:
        gold, meta, model, batch = build_case("pase_plus_workers_3200", "cuda")
        model.frontend.precision = precision
        runs = []
        for _ in range(2):
            random.seed(meta["seed"])
            torch.manual_seed(meta["seed"])
            model.zero_grad(set_to_none=True)
            h, chunk, preds, labels = model(batch, 1, "cuda")
            tot, _ = total_loss(model, preds, labels)
            tot.backward()
            runs.append((tot.detach().clone(),
                         {k: p.grad.clone() for k, p in model.named_parameters()}))
    finally:
        Fn.set_precision(prev)
    (t1, g1), (t2, g2) = runs
    assert torch.equal(t1, t2), (float(t1), float(t2))
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_mlp_minion_accepts_reference_layout_tensors():
    """A (B,C,T) tensor that did not come from the encoder goes through the NCT->rows kernel."""
    torch.manual_seed(0)
    m = MLPMinion(num_inputs=64, num_outputs=5, dropout=0, hidden_size=32, hidden_layers=1,
                  r=3, skip=False, loss=ContextualizedLoss("MSELoss", 3)).cuda()
    x = torch.randn(2, 64, 17, device="cuda", requires_grad=True)
    lab = torch.randn(2, 5, 17, device="cuda")
    y = m(x)
    assert tuple(y.shape) == (2, 15, 17)
    loss = m.loss(y, lab)
    loss.backward()
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    xc = x.detach().cpu().requires_grad_(True)
    yr = O.head_mlp(xc, sd, "", 1)
    lr = ((yr - O.contextualize(lab.cpu(), 3)) ** 2).mean()
    lr.backward()
    assert_close(y, yr, 1e-4, 1e-5, "mlp pred")
    assert_close(loss, lr, 1e-4, 1e-6, "ctx mse")
    assert_close(x.grad, xc.grad, 1e-3, 1e-6, "dx")


def test_spc_worker_runs_and_matches_oracle_math():
    import random
    from pase_b200.minions import cls_worker_maker
    cfg = {"num_outputs": 1, "dropout": 0, "hidden_size": 32, "hidden_layers": 1, "name": "spc",
           "type": "spc", "loss": ContextualizedLoss("BCEWithLogitsLoss"), "skip": False}
    torch.manual_seed(1)
    w = cls_worker_maker(cfg, 20).cuda()
    x = torch.randn(3, 20, 100, device="cuda")
    random.seed(5)
    y, lab = w(x, 1, device="cuda")
    assert tuple(y.shape) == (6, 1, 1) and tuple(lab.shape) == (6, 1, 1)
    loss = w.loss(y, lab)
    # same draws on the CPU
    random.seed(5)
    N, M = 5, 21
    T = 100
    t = random.choice(list(range(M + 1, T - M)))
    ft = random.choice(list(range(t + 16, T - N)))
    pt = random.choice(list(range(N, t - 16)))
    xc = x.cpu()
    fut, past, cur = xc[:, :, ft:ft + N].reshape(3, -1), xc[:, :, pt - N:pt].reshape(3, -1), xc[:, :, t]
    full = torch.cat([torch.cat([cur, fut], 1), torch.cat([cur, past], 1)], 0).unsqueeze(2)
    sd = {k[len("minion."):]: v.detach().cpu() for k, v in w.state_dict().items()}
    yr = O.head_mlp(full, sd, "", 1)
    assert_close(y, yr, 1e-4, 1e-5, "spc logits")
    ref = torch.nn.functional.binary_cross_entropy_with_logits(
        yr, torch.cat([torch.ones(3, 1, 1), torch.zeros(3, 1, 1)], 0))
    assert_close(loss, ref, 1e-4, 1e-6, "spc bce")


def _workers_plus_cfg():
    mlp = lambda name, nout: {"num_outputs": nout, "dropout": 0, "hidden_size": 256,
                              "hidden_layers": 1, "name": name, "context": 1, "r": 7,
                              "loss": "MSELoss", "skip": False}
    regr = [{"num_outputs": 1, "dropout": 0, "dropout_time": 0.0, "hidden_layers": 1,
             "name": "cchunk", "type": "decoder", "hidden_size": 64, "fmaps": [512, 256, 128],
             "strides": [4, 4, 10], "kwidths": [30, 30, 30], "loss": "L1Loss"}]
    for name, nout in (("lps", 3075), ("lps_long", 3075), ("fbank", 120), ("fbank_long", 120),
                       ("gtn", 120), ("gtn_long", 120), ("mfcc", 39), ("mfcc_long", 60),
                       ("prosody", 12)):
        regr.append(mlp(name, nout))
    cls = [{"num_outputs": 1, "dropout": 0, "hidden_size": 256, "hidden_layers": 1, "name": n,
            "loss": "BCEWithLogitsLoss", "skip": False, "augment": n == "cmi"}
           for n in ("mi", "cmi")]
    return {"regr": regr, "cls": cls}


@pytest.mark.parametrize("precision", ["3xf16", "3xtf32"])
def test_workers_plus_full_length_against_oracle(precision):
    """BASELINE.json configs[2]/[3] model (PASE+.cfg + all 12 workers+ heads) at the real
    chunk length T=32000 (T'=200), B=4 chunk triplets: every loss and the summed loss against
    the CPU oracle (fp32 bar), every parameter gradient in relative L2 (the L1-driven decoder
    path, sign(pred-target), only through its norm)."""
    import copy
    from helpers import resolve_cfg, fill_state_dict, rel_l2
    from pase_b200.pase import pase as native_pase, total_loss
    from pase_b200.utils import parse_workers
    from pase_b200 import functional as Fn
    fe_cfg, wcfg = resolve_cfg("cfg/frontend/PASE+.cfg"), _workers_plus_cfg()
    B, T, Tq, seed = 4, 32000, 200, 71
    prev = Fn.PRECISION
    Fn.set_precision(precision)
    try:
        model = native_pase(frontend_cfg=fe_cfg, minions_cfg=parse_workers(copy.deepcopy(wcfg)))
        sd = fill_state_dict(model.state_dict(), seed)
        model.load_state_dict(sd)
        model.frontend.precision = precision
        model = model.cuda().train()
        batch = {k: seeded_randn((B, 1, T), seed + 10 + i, 0.5)
                 for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
        for i, w in enumerate(wcfg["regr"]):
            if w["name"] != "cchunk":
                batch[w["name"]] = seeded_randn((B, w["num_outputs"], Tq), seed + 100 + i)
        leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()
                  if v.is_floating_point() and "running" not in k}
        full = dict(sd)
        full.update(leaves)
        _, chunk_r, preds_r, labels_r = O.pase_forward(batch, full, fe_cfg, wcfg, training=True)
        tot_r, per_r = O.total_loss(preds_r, labels_r, wcfg)
        tot_r.backward()
        h, chunk, preds, labels = model({k: v.cuda() for k, v in batch.items()}, 1, "cuda")
        assert_close(chunk, chunk_r, 1e-3, 1e-5, "chunk")
        tot, per = total_loss(model, preds, labels)
        for k, v in per.items():
            assert_close(v, per_r[k], 2e-4, 1e-6, "loss " + k)
        assert_close(tot, tot_r, 2e-4, 1e-6, "total")
        assert tuple(preds["lps"].shape) == (B, 21525, Tq)
        tot.backward()
        bad = []
        for k, p in model.named_parameters():
            ref = leaves[k].grad
            if k.startswith("frontend.") and (k.endswith("conv.bias") or k.endswith("W.bias")):
                continue                                  # analytically zero under train-mode BN
            r = rel_l2(p.grad.cpu(), ref)
            # the L1-driven decoder path (sign(pred - target)) feeds every frontend gradient
            lim = 2e-2 if (k.startswith(("regression_workers.0.", "frontend.")) or "_hz_" in k) \
                else 3e-3
            if r >= lim:
                bad.append("%s %.2e" % (k, r))
        assert not bad, "; ".join(bad[:10])
    finally:
        Fn.set_precision(prev)


def test_fused_regression_heads_gpu():
    """pase.fuse_regression_loss on the GPU (3xF16): the contextualised-MSE epilogue of the
    output GEMM gives the same losses and gradients as the unfused heads at T=32000, and the
    fused GEMM kernel matches its spec (tests/emul/heads.py) on a ragged shape."""
    import copy
    import emul
    from pase_b200 import _lib
    from helpers import resolve_cfg, fill_state_dict, rel_l2
    from pase_b200.pase import pase as native_pase, total_loss
    from pase_b200.utils import parse_workers
    from pase_b200 import functional as Fn
    # --- kernel vs spec: B=3, T=50, F=11, r=7 (N=77 -> ldr=128), K=128
    B, T, F, r, K = 3, 50, 11, 7, 128
    M, N, ldr = B * T, F * r, 128
    g = torch.Generator().manual_seed(5)
    h = torch.randn(M * K, generator=g)
    W = torch.randn(N * K, generator=g) * 0.1
    bias, label = torch.randn(N, generator=g), torch.randn(B * F * T, generator=g)
    def pair(x):
        hi = x.to(torch.float16)
        return hi, ((x - hi.float()) * 2048.0).to(torch.float16)
    (hh, hl), (wh, wl) = pair(h), pair(W)
    scale = torch.tensor([1.0 / 64.0, 64.0])
    args = [hh, hl, M, K, wh, wl, K, torch.zeros(M * ldr, dtype=torch.float16),
            torch.zeros(M * ldr, dtype=torch.float16), ldr, M, N, K, bias, label, B, F, T, r, scale,
            torch.zeros(1, dtype=torch.float64), torch.zeros(ldr, dtype=torch.float64)]
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul.call("pase_tc_gemm_nt_ctxmse", *cpu)
    _lib.call("pase_tc_gemm_nt_ctxmse", *dev)
    torch.cuda.synchronize()
    vc = cpu[7].float() + cpu[8].float() / 2048.0
    vd = dev[7].cpu().float() + dev[8].cpu().float() / 2048.0
    assert float((vc - vd).abs().max()) <= 4e-6 * float(vc.abs().max())
    assert abs(float(cpu[20]) - float(dev[20].cpu())) <= 1e-5 * float(cpu[20])
    assert float((cpu[21] - dev[21].cpu()).abs().max()) <= 1e-5 * float(cpu[21].abs().max())
    # --- whole model, fused vs unfused
    fe_cfg, wcfg = resolve_cfg("cfg/frontend/PASE+.cfg"), _workers_plus_cfg()
    Bm, Tm, Tq, seed = 2, 32000, 200, 73
    prev = Fn.PRECISION
    Fn.set_precision("3xf16")
    try:
        res = {}
        for fused in (False, True):
            model = native_pase(frontend_cfg=fe_cfg, minions_cfg=parse_workers(copy.deepcopy(wcfg)))
            model.load_state_dict(fill_state_dict(model.state_dict(), seed))
            model = model.cuda().train()
            model.fuse_regression_loss = fused
            batch = {k: seeded_randn((Bm, 1, Tm), seed + 10 + i, 0.5).cuda()
                     for i, k in enumerate(["chunk", "chunk_ctxt", "chunk_rand", "cchunk"])}
            for i, w in enumerate(wcfg["regr"]):
                if w["name"] != "cchunk":
                    batch[w["name"]] = seeded_randn((Bm, w["num_outputs"], Tq), seed + 100 + i).cuda()
            hh_, chunk, preds, labels = model(batch, 1, "cuda")
            tot, per = total_loss(model, preds, labels)
            tot.backward()
            res[fused] = (float(tot), {k: float(v) for k, v in per.items()},
                          {k: p.grad.detach().cpu() for k, p in model.named_parameters()})
        (ta, la, ga), (tb, lb, gb) = res[False], res[True]
        assert abs(ta - tb) <= 2e-5 * abs(ta)
        for k in la:
            assert abs(la[k] - lb[k]) <= 5e-5 * max(abs(la[k]), 1e-6), k
        for k in ga:
            if k.startswith("regression_workers") and not k.startswith("regression_workers.0."):
                # the fused heads themselves.  The two models' encoder outputs differ by ~4e-7
                # (order of the BatchNorm statistics' atomics), which now and then flips ONE
                # hidden PReLU gate of a head (|u| ~ 1e-7): the hidden layer's weight / bias
                # gradients then move by ~(1-alpha) dh x^T / |dW| = 2e-4..1e-3 (measured; the
                # same spread shows between two unfused runs).  Output-layer gradients have no
                # gate between them and the loss.
                lim = 5e-3 if ".blocks." in k and ".W." in k else 2e-5
                assert rel_l2(gb[k], ga[k]) < lim, (k, rel_l2(gb[k], ga[k]))
    finally:
        Fn.set_precision(prev)
