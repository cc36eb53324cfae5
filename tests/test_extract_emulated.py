"""Host side of WaveFe.extract (packed variable-length inference) on CPU, every kernel launch
replaced by its torch emulation (tests/emul/): the planner's offsets and table, the
packed forward against the eval goldens and the per-utterance forward, capacity splitting,
the 32-bit index guard and a launch count independent of the number of utterances."""
import pytest
import torch

import emul
from helpers import load_golden, resolve_cfg, fill_state_dict, seeded_randn, assert_close
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import EXTRACT_MAX_SAMPLES, WaveFe


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    yield


def make_model(cfg_name, precision, seed=11):
    model = WaveFe(**resolve_cfg(cfg_name))
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    return model.eval()


def single(model, x):
    """B=1 forward of one utterance with the emulated uniform kernels."""
    model._sinc_consts(x.device)
    plan = model._plan(1, x.numel(), x.device)
    with torch.no_grad():
        y, _ = enc.encoder_forward(plan, model, x.view(1, 1, -1), dict(model.named_parameters()),
                                   False, False)
    return y


@pytest.mark.parametrize("precision", ["fp32", "3xtf32", "3xf16"])
@pytest.mark.parametrize("name", ["enc_pase_eval_16000", "enc_pasep_eval_3200"])
def test_packed_matches_goldens_and_single(name, precision, emulated):
    gold, meta = load_golden(name)
    model = WaveFe(**resolve_cfg(meta["cfg"]))
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), meta["seed"]))
    model.eval()
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    others = [seeded_randn((T,), 50 + T, 0.5) for T in (471, 1763, 2345)]
    wavs = [others[0], x[0, 0], others[1]] + [x[n, 0] for n in range(1, meta["N"])] + [others[2]]
    feats = model._extract(wavs, None, None, torch.device("cpu"))
    assert len(feats) == len(wavs)
    golden_idx = [1] + list(range(3, 3 + meta["N"] - 1))
    for n, i in enumerate(golden_idx):
        assert_close(feats[i][0], gold["y"][n], 1e-4, 1e-5, "%s utt %d" % (name, i))
    for i in (0, 2, len(wavs) - 1):
        assert_close(feats[i], single(model, wavs[i]), 1e-4, 1e-5, "single %d" % i)


def test_layout_alignment_and_separator_rows(emulated):
    model = make_model("cfg/frontend/PASE+.cfg", "3xf16")
    lengths = [3200, 471, 4001, 1000]
    wavs = [seeded_randn((T,), T, 0.5) for T in lengths]
    plan = model._packed_plan(enc.min_length(model.cfg) * 8 + sum(lengths), torch.device("cpu"))
    geoms = enc.utterance_geometry(model.cfg, lengths, plan.precision.sinc_fold)
    host, sec, sz = enc.packed_layout(plan, lengths, geoms, None)
    n, G = len(lengths), plan.geoms
    wave = host[sec["wave"]:sec["wave"] + 3 * n].view(n, 3)
    assert (wave[:, 2] % G[0].lda == 0).all()                 # fold-aligned sinc operand
    for l, g in enumerate(G):
        bn = host[sec[("bn", l)]:sec[("bn", l)] + 6 * n].view(n, 6)
        gm = host[sec[("gemm", l)]:sec[("gemm", l)] + 3 * n + 1]
        assert gm[:n + 1].tolist() == [0] + torch.cumsum(
            torch.tensor([gi[l].P for gi in geoms]), 0).tolist()
        assert gm[2 * n + 1:].tolist() == [gi[l].T_out for gi in geoms]
        if l + 1 < len(G):
            assert (bn[:, 2] % G[l + 1].lda == 0).all()       # stride-aligned conv operand
            nxt = host[sec[("gemm", l + 1)]:sec[("gemm", l + 1)] + n]
            assert (bn[:, 2] // G[l + 1].lda == nxt).all()
    # separator rows of the QRNN input: poisoned before the call, zero after it
    plan.xq.fill_(3.0)
    model._sinc_consts(torch.device("cpu"))
    feats = enc.encoder_forward_packed(plan, model, torch.cat(wavs), lengths, geoms,
                                       dict(model.named_parameters()))
    Cq = plan.Clast
    xr = [0]
    for gi in geoms:
        xr.append(xr[-1] + gi[-1].T_out + 1)
    for i in range(n):
        assert (plan.xq[xr[i] * Cq:(xr[i] + 1) * Cq] == 0).all()
    for i, w in enumerate(wavs):
        assert_close(feats[i], single(model, w), 1e-4, 1e-5, "utt %d" % i)


def test_split_packs():
    assert enc.split_packs([], 10) == []
    assert enc.split_packs([4, 4, 4], 8) == [(0, 2), (2, 3)]
    assert enc.split_packs([4, 20, 4], 8) == [(0, 1), (1, 2), (2, 3)]
    assert enc.split_packs([3, 3, 3, 3], 100) == [(0, 4)]


def test_capacity_split_matches_one_pack(emulated):
    model = make_model("cfg/frontend/PASE+.cfg", "fp32")
    wavs = [seeded_randn((T,), T, 0.5) for T in (1000, 3200, 471, 2500, 1763)]
    ref = model._extract(wavs, "avg_norm", None, torch.device("cpu"))
    split = model._extract(wavs, "avg_norm", 3000, torch.device("cpu"))    # 3200 > cap
    assert sorted(k[0] for k in model._packed_plans) == [3000, 3200, EXTRACT_MAX_SAMPLES]
    assert [tuple(f.shape) for f in split] == [tuple(f.shape) for f in ref]
    for a, b in zip(split, ref):
        assert_close(a, b, 1e-5, 1e-6, "split")
    y = single(model, wavs[1])
    assert_close(split[1], y - y.mean(2, keepdim=True), 1e-4, 1e-5, "avg_norm")


def test_index_guard():
    cfg = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    with pytest.raises(ValueError, match="32-bit"):
        enc.PackedPlan(cfg, 40_000_000, torch.device("meta"), "3xf16")
    plan = enc.PackedPlan(cfg, 1 << 21, torch.device("meta"), "3xf16")
    assert max(t.numel() for t in plan.tensors()) < enc.INDEX_LIMIT


def test_launches_independent_of_utterance_count(emulated, monkeypatch):
    model = make_model("cfg/frontend/PASE+.cfg", "3xf16")
    counts = []
    for n in (4, 40):
        wavs = [seeded_randn((471 + 37 * i,), i, 0.5) for i in range(n)]
        calls = []
        monkeypatch.setattr(ops, "call", lambda name, *a: (calls.append(name),
                                                           emul.call(name, *a))[1])
        model._extract(wavs, "avg_concat", None, torch.device("cpu"))
        counts.append(calls)
    assert counts[0] == counts[1]


def test_argument_errors(emulated, monkeypatch):
    model = make_model("cfg/frontend/PASE+.cfg", "3xf16")
    calls = []
    monkeypatch.setattr(ops, "call", lambda name, *a: calls.append(name))
    assert model._extract([], None, None, torch.device("cpu")) == []
    with pytest.raises(ValueError, match="utterance 1 .*block"):
        model._extract([torch.zeros(1000), torch.zeros(470)], None, None, torch.device("cpu"))
    with pytest.raises(ValueError, match="utterance 0"):
        model._extract([torch.zeros(2, 1000)], None, None, torch.device("cpu"))
    with pytest.raises(TypeError, match="utterance 0"):
        model._extract([torch.zeros(1000, dtype=torch.float64)], None, None, torch.device("cpu"))
    with pytest.raises(ValueError, match="mode"):
        model._extract([torch.zeros(1000)], "avg", None, torch.device("cpu"))
    with pytest.raises(RuntimeError, match="CUDA"):
        model.extract([torch.zeros(1000)])
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        model.extract([torch.zeros(1000)])
    assert calls == []
    assert enc.min_length(model.cfg) == 471
