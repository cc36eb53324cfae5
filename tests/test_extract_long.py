"""Host side of WaveFe.extract_long / FeatureStream (windowed inference of one long recording)
on CPU, every kernel launch replaced by its torch emulation (tests/emul/): the window
planner, the halos it derives against the float64 oracle, the windowed forward against the
B=1 forward, the stream against extract_long, and argument errors raised before any launch."""
import random

import pytest
import torch
import torch.nn.functional as F

import emul
import pase_oracle as O
from helpers import resolve_cfg, fill_state_dict, seeded_randn, assert_close
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import FeatureStream, WaveFe

CFGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
CPU = torch.device("cpu")


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    yield


def make_model(cfg_name, precision="fp32", seed=11):
    model = WaveFe(**resolve_cfg(cfg_name))
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    return model.eval()


def single(model, x):
    model._sinc_consts(x.device)
    plan = model._plan(1, x.numel(), x.device)
    with torch.no_grad():
        y, _ = enc.encoder_forward(plan, model, x.view(1, 1, -1), dict(model.named_parameters()),
                                   False, False)
    return y


def _check_plan(cfg, L, window):
    hop, segs = enc.hop_size(cfg), enc.plan_windows(cfg, L, window)
    T = enc.frame_counts(cfg, L)[-1]
    frames = []
    for k, sg in enumerate(segs):
        s, n = sg["seg_start"], sg["seg_len"]
        assert s % hop == 0 and n >= enc.min_length(cfg)
        assert n <= enc.window_capacity(cfg, window)
        if cfg["denseskips"] and not (s == 0 and s + n == L):
            assert enc.pool_factors(cfg, n) == enc.nominal_pool_factors(cfg)
        first = s // hop + sg["crop_f0"]
        frames += list(range(first, first + sg["crop_n"]))
    assert segs[0]["seg_start"] == 0
    assert segs[-1]["seg_start"] + segs[-1]["seg_len"] == L
    assert frames == list(range(T))
    if cfg["denseskips"]:
        assert enc.pool_factors(cfg, L) == enc.nominal_pool_factors(cfg)
    return segs


@pytest.mark.parametrize("cfg_name", CFGS)
def test_stream_planner_tiles_the_frames(cfg_name):
    cfg = WaveFe(**resolve_cfg(cfg_name)).cfg
    hop, w = enc.hop_size(cfg), enc.min_window(cfg)
    assert hop == 160 and w == 81920
    assert enc.receptive_field(cfg) == (1034, 1335)
    assert enc.window_halos(cfg) == ((8 if cfg["rnn_pool"] else 7), 8)
    for r in (0, 1, 77):
        for L in (w + 1 * hop + r, 3 * w + 977 * hop + r, 7 * w + r):
            _check_plan(cfg, L, w)
        _check_plan(cfg, 5 * w + 300 * hop + r, 2 * w + 3 * hop)
    segs = _check_plan(cfg, w + hop, w)                    # T' = 513: a short last crop
    assert segs[-1]["crop_n"] == 513 - enc.final_frames(cfg, w)
    segs = _check_plan(cfg, 2 * w + 160 * 20 + 5, w)        # a short tail, extended left
    assert segs[-1]["seg_len"] >= enc.tail_length(cfg)
    with pytest.raises(ValueError, match="window"):
        enc.plan_windows(cfg, 10 * w, w - hop)
    L = 3 * w + 159                                         # T' = ceil(L/160): d_0 = 159
    if cfg["denseskips"]:
        assert enc.pool_factors(cfg, L)[0] == 159
        with pytest.raises(NotImplementedError, match="pools its dense skips"):
            enc.plan_windows(cfg, L, w)
    else:
        _check_plan(cfg, L, w)


def test_tail_length_is_minimal():
    cfg = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    tail = enc.tail_length(cfg)
    assert enc.pool_factors(cfg, tail) == enc.nominal_pool_factors(cfg)
    assert enc.pool_factors(cfg, tail - 160) != enc.nominal_pool_factors(cfg)
    assert enc.pool_factors(cfg, 7597)[0] == 161


def _pre_qrnn(x, sd, cfg):
    """Float64 oracle: the QRNN input and the pooled dense skips, (C + emb*, T')."""
    c = dict(cfg, rnn_pool=False)
    _, blocks = O.encoder_forward(x.view(1, 1, -1), sd, c, training=False, return_blocks=True)
    Tq = blocks[-1].shape[2]
    parts = [blocks[-1]]
    for i in range(len(blocks) - 1):
        parts.append(O._pool_skip(F.conv1d(blocks[i], sd["denseskips.%d.weight" % i]), Tq))
    return torch.cat(parts, 1)[0]


def test_derived_halos_against_oracle():
    cfg = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    sd = {k: v.double() for k, v in
          fill_state_dict(WaveFe(**cfg).state_dict(), 11).items() if v.is_floating_point()}
    hop = enc.hop_size(cfg)
    x = seeded_randn((64000,), 3, 0.5).double()
    whole = _pre_qrnn(x, sd, cfg)
    hl, hr = enc.window_halos(cfg)
    hl -= 1                                   # the part before the QRNN: no x_{t-1}
    f0, f1 = 100, 260

    def crop(left, right):
        s, e = (f0 - left) * hop, (f1 + right) * hop
        return _pre_qrnn(x[s:e], sd, cfg)[:, left:left + f1 - f0], whole[:, f0:f1]

    got, ref = crop(hl, hr)
    assert float((got - ref).abs().max()) < 1e-10         # float64 rounding
    got, ref = crop(hl - 1, hr)
    assert float((got[:, 0] - ref[:, 0]).abs().max()) > 2e-5
    got, ref = crop(hl, hr - 1)
    assert float((got[:, -1] - ref[:, -1]).abs().max()) > 2e-5


@pytest.mark.parametrize("cfg_name", CFGS)
def test_pooled_extract_long_matches_single(cfg_name, emulated):
    model = make_model(cfg_name)
    w = enc.min_window(model.cfg)
    x = seeded_randn((w + 160 * 30 + 77,), 21, 0.5)
    got = model._extract_long(x, None, w, CPU)
    assert len(enc.plan_windows(model.cfg, x.numel(), w)) == 2
    assert_close(got, single(model, x), 1e-4, 1e-5, cfg_name)
    y = got
    for mode in ("avg_norm", "avg_concat", "avg_norm_concat"):
        g = model._extract_long(x, mode, w, CPU)
        ref = O.select_output(y, mode)
        assert g.shape == ref.shape
        assert float((g - ref).abs().max()) <= 1e-6 * float(y.abs().max()), mode


def test_pooled_stream_matches_extract_long(emulated):
    model = make_model("cfg/frontend/PASE+.cfg")
    cfg = model.cfg
    w = enc.min_window(cfg)
    x = seeded_randn((w + 160 * 40 + 1,), 22, 0.5)
    ref = model._extract_long(x, None, w, CPU)
    rng = random.Random(3)
    for trial in range(2):
        st = FeatureStream(model, CPU, w)
        outs, a = [], 0
        while a < x.numel():
            n = rng.choice([1, 160, 1000, rng.randrange(1, 40000)])
            y = st.push(x[a:a + n])
            a = min(a + n, x.numel())
            assert y.shape[2] == enc.final_frames(cfg, a) - sum(o.shape[2] for o in outs)
            outs.append(y)
        outs.append(st.finish())
        got = torch.cat(outs, 2)
        assert got.shape == ref.shape
        assert_close(got, ref, 1e-5, 1e-6, "trial %d" % trial)
        with pytest.raises(RuntimeError, match="after finish"):
            st.push(x[:10])


def test_argument_errors_before_any_segment(emulated, monkeypatch):
    model = make_model("cfg/frontend/PASE+.cfg", "3xf16")
    w = enc.min_window(model.cfg)
    calls = []
    monkeypatch.setattr(ops, "call", lambda name, *a: calls.append(name))
    with pytest.raises(ValueError, match="window"):
        model._extract_long(torch.zeros(3 * w), None, w - 1, CPU)
    with pytest.raises(ValueError, match="recording"):
        model._extract_long(torch.zeros(2, w), None, w, CPU)
    with pytest.raises(TypeError):
        model._extract_long(torch.zeros(w, dtype=torch.float64), None, w, CPU)
    with pytest.raises(ValueError, match="mode"):
        model._extract_long(torch.zeros(3 * w), "avg", w, CPU)
    with pytest.raises(NotImplementedError):
        model._extract_long(torch.zeros(3 * w + 155), None, w, CPU)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.extract_long(torch.zeros(3 * w))
    with pytest.raises(RuntimeError, match="CUDA"):
        model.stream()
    st = FeatureStream(model, CPU, w)
    assert st.push(torch.zeros(300)).shape == (1, model.emb_dim, 0)
    assert calls == ["pase_stream_gather"]                # the samples go to the stream's ring
    del calls[:]
    with pytest.raises(ValueError, match="shorter"):
        st.finish()
    with pytest.raises(ValueError, match="window"):
        FeatureStream(model, CPU, w - 160)
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        model.extract_long(torch.zeros(3 * w))
    with pytest.raises(RuntimeError, match="eval"):
        model.stream()
    with pytest.raises(RuntimeError, match="eval"):
        st.push(torch.zeros(10))
    assert calls == []
