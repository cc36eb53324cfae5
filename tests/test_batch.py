"""On-device batch assembly (pase_b200/batch.py, pase_b200/csrc/batch.cu), CPU side.

The planner reproduces the reference's draw streams and the emulated pipeline reproduces the
reference's collated batches bit for bit (tests/golden/batch.pt, made by make_batch_golden.py
from the unmodified reference), the neighbour lists behave as the reference's across batches
and epochs, every refusal names what it refuses, the pools pack the corpus as documented, and
from_train_opts builds the workers+ recipe.
"""
import json
import os
import pickle
import random

import numpy as np
import pytest
import torch

import emul
from batch_corpus import CASES, HOP, KEYS, SPLIT, T, UTTS, build_corpus, digest
from distortion_banks import build_banks, case_cfg
from helpers import GOLDEN
from make_batch_golden import BatchRecorder
from pase_b200 import ops
from pase_b200.batch import DeviceBatcher, FeaturePool, WavPool
from pase_b200.distortions import config_distortions

# the workers+ recipe (cfg/workers/workers+.cfg): names and transform overrides, in cfg order
WORKERS_PLUS = {
    "regr": [{"name": "cchunk"}, {"name": "lps"}, {"name": "lps_long", "transform": {"win": 512}},
             {"name": "fbank"}, {"name": "fbank_long", "transform": {"win": 1024, "n_fft": 1024}},
             {"name": "gtn"}, {"name": "gtn_long", "transform": {"win": 2048}},
             {"name": "mfcc"}, {"name": "mfcc_long", "transform": {"win": 2048, "order": 20}},
             {"name": "prosody"}],
    "cls": [{"name": "mi"}, {"name": "cmi"}],
}
PLUS_KEYS = {"fbank": 120, "fbank_long": 120, "gtn": 120, "gtn_long": 120, "mfcc": 39,
             "mfcc_long": 60, "prosody": 12}


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("batch_corpus"))
    data_root, cfg, cache = build_corpus(root)
    banks = build_banks(os.path.join(root, "banks"))
    return dict(root=root, data_root=data_root, cfg=cfg, cache=cache, banks=banks)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "batch.pt"))


def _pool(corpus):
    return WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement="cpu")


def _batcher(corpus, case, wavs=None, device="cpu", placement="cpu"):
    c = CASES[case]
    wavs = wavs or WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement=placement)
    cached = None
    if c["cached"]:
        cached = {k: (FeaturePool(corpus["cache"], SPLIT, k, wavs.names, placement), HOP)
                  for k in KEYS}
    dist = None
    if c["distortions"]:
        dist = config_distortions(device=device, **case_cfg("pase_plus", corpus["banks"])[0])
    return DeviceBatcher(wavs, T, mi=c["mi"], random_scale=c["random_scale"], cached=cached,
                         distortions=dist)


def _seed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def _meta(golden, case):
    return json.loads(golden[case + "/meta"])


def _normalise(log, index, n):
    """The planner draws the random utterance as choice(range(n - 1)) -> j; the reference
    draws from the index list without `index` -> j + (j >= index)."""
    out = []
    for ev in log:
        if ev[0] == "choice" and ev[1] == n - 1 and isinstance(ev[2], int):
            ev = ["choice", ev[1], ev[2] + (ev[2] >= index)]
        out.append(ev)
    return out


# ------------------------------------------------------------------------------ planner


@pytest.mark.parametrize("case", list(CASES))
def test_planner_reproduces_reference_draws(case, corpus, golden):
    meta = _meta(golden, case)
    b = _batcher(corpus, case)
    n = len(UTTS)
    _seed(CASES[case]["seed"])
    k = 0
    for idx in CASES[case]["batches"]:
        for i in idx:
            with BatchRecorder() as rec:
                s = b._draw(i, random, np.random, None)
            want = meta["samples"][k]
            assert (s["index"], s["ctxt"], s["rand"], s["beg"]) == \
                (want["index"], want["ctxt"], want["rand"], want["beg"]), (case, k)
            if want["scale"] is None:
                assert s["scale"] is None
            else:
                assert np.array_equal(np.float32(s["scale"]), np.float32(want["scale"]))
            assert _normalise(rec.log, i, n) == meta["logs"][k], (case, k)
            k += 1
    assert k == len(meta["samples"])


def test_plan_with_explicit_generators_matches_globals(corpus):
    b = _batcher(corpus, "mi_dist")
    _seed(5)
    p1 = b.plan([3, 6, 12])
    b.reset()
    g = torch.Generator()
    g.manual_seed(5)
    p2 = b.plan([3, 6, 12], rng=(random.Random(5), np.random.RandomState(5), g))
    assert np.array_equal(p1.table, p2.table)
    assert p1.samples == p2.samples


# ------------------------------------------------------------------------------ pipeline


def _check_batch(out, want, case, dist_chunk=None):
    assert set(out) == set(want) | ({"chunk"} if dist_chunk is not None else set())
    for k, w in want.items():
        a = out[k].cpu().numpy()
        assert list(a.shape) == w["shape"], (case, k)
        assert digest(a) == w["sha256"], (case, k)
    if dist_chunk is not None:
        y = out["chunk"].cpu().double().reshape(dist_chunk.shape[0], -1).numpy()
        ref = dist_chunk.double().reshape(y.shape[0], -1).numpy()
        for r in range(y.shape[0]):
            rel = np.linalg.norm(y[r] - ref[r]) / max(np.linalg.norm(ref[r]), 1e-30)
            mx = np.abs(y[r] - ref[r]).max() / max(np.abs(ref[r]).max(), 1e-30)
            assert rel < 3e-6 and mx < 1e-5, (case, r, rel, mx)


@pytest.mark.parametrize("case", list(CASES))
def test_emulated_pipeline_matches_golden_hashes(case, corpus, golden, monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    meta = _meta(golden, case)
    b = _batcher(corpus, case)
    _seed(CASES[case]["seed"])
    for bi, idx in enumerate(CASES[case]["batches"]):
        out = b(idx)
        _check_batch(out, meta["arrays"][bi], case, golden.get("%s/%d/chunk" % (case, bi)))


def test_silent_chunk_scales_to_nan(corpus, monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    b = _batcher(corpus, "single_short")
    out = b([9])
    assert bool(torch.isnan(out["chunk"]).all()) and bool(torch.isnan(out["cchunk"]).all())


def test_short_utterance_is_reflect_padded(corpus, monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    wavs = _pool(corpus)
    b = DeviceBatcher(wavs, T, mi=False)
    out = b([4])
    u = wavs.samples(4)
    L = len(u)
    want = torch.nn.functional.pad(torch.from_numpy(u).view(1, 1, -1), (0, T - L),
                                   mode="reflect").view(-1)
    assert torch.equal(out["chunk"].view(-1), want)


# ------------------------------------------------------------------------------ reset


def test_neighbour_lists_shrink_and_reset_restores_them(corpus):
    b = _batcher(corpus, "mi_short")
    _seed(1)
    b.plan([0, 1, 2])
    # 1001-134707-0001-* has 4 segments; after visiting 0, 1, 2 only segment 3 is left
    assert b._neighbors["1001-134707-0001-"] == ["1001-134707-0001-3.wav"]
    with BatchRecorder() as rec:
        s = b._draw(3, random, np.random, None)
    assert s["ctxt"] == 3                      # empty list: the utterance itself, no draw
    assert [ev[0] for ev in rec.log[:2]] == ["random", "choice"] and rec.log[1][1] == len(UTTS) - 1
    with pytest.raises(ValueError, match="visited twice"):
        b.plan([2])
    b.reset()
    _seed(1)
    p = b.plan([0, 1, 2])
    assert len(p.samples) == 3


# ------------------------------------------------------------------------------ refusals


def test_refusals_name_what_they_refuse(corpus, tmp_path):
    wavs = _pool(corpus)
    with pytest.raises(NotImplementedError, match="zero_speech_p"):
        DeviceBatcher(wavs, T, zero_speech_p=0.1)
    fb = FeaturePool(corpus["cache"], SPLIT, "fbank", wavs.names, "cpu")
    with pytest.raises(ValueError, match="'fbank'.*hop 160"):
        DeviceBatcher(wavs, 4001, cached={"fbank": (fb, HOP)})
    # a padded chunk has fewer frames than the slice needs
    b = DeviceBatcher(wavs, T, mi=False, cached={"fbank": (fb, HOP)})
    with pytest.raises(ValueError, match="'fbank'.*1001-134707-0002-0.wav"):
        b.plan([4])
    # reflect padding of P >= L samples
    b = DeviceBatcher(wavs, 6000, mi=False)
    with pytest.raises(ValueError, match="1001-134707-0002-0.wav.*2500 samples"):
        b.plan([4])
    # one utterance: no random utterance to draw
    one = os.path.join(str(tmp_path), "one.json")
    cfg = json.load(open(corpus["cfg"]))
    cfg[SPLIT]["data"] = cfg[SPLIT]["data"][:1]
    json.dump(cfg, open(one, "w"))
    with pytest.raises(ValueError, match="at least 2"):
        DeviceBatcher(WavPool(corpus["data_root"], one, SPLIT, placement="cpu"), T)
    b = DeviceBatcher(wavs, T)
    with pytest.raises(ValueError, match="index 13 outside"):
        b.plan([13])


def test_feature_pool_refusals(corpus, tmp_path):
    wavs = _pool(corpus)
    cache = str(tmp_path)
    d = os.path.join(cache, SPLIT, "gtn")
    os.makedirs(d)
    bases = [os.path.splitext(n)[0] for n in wavs.names]
    for i, bname in enumerate(bases[:-1]):
        torch.save(torch.zeros(3, 10), os.path.join(d, bname + ".gtn"))
    with pytest.raises(ValueError, match="5005-4-0007-0.gtn is missing"):
        FeaturePool(cache, SPLIT, "gtn", wavs.names, "cpu")
    torch.save(torch.zeros(3, 10, dtype=torch.float64), os.path.join(d, bases[-1] + ".gtn"))
    with pytest.raises(ValueError, match="5005-4-0007-0.gtn.*float64"):
        FeaturePool(cache, SPLIT, "gtn", wavs.names, "cpu")
    torch.save(torch.zeros(4, 10), os.path.join(d, bases[-1] + ".gtn"))
    with pytest.raises(ValueError, match="5005-4-0007-0.gtn has F=4, the first file has F=3"):
        FeaturePool(cache, SPLIT, "gtn", wavs.names, "cpu")


def test_wav_pool_refuses_other_formats(corpus, tmp_path):
    from scipy.io import wavfile
    root = str(tmp_path)
    wavfile.write(os.path.join(root, "a-1-1-0.wav"), 16000, np.zeros(100, np.int16))
    wavfile.write(os.path.join(root, "a-1-1-1.wav"), 16000, np.zeros(100, np.int32))
    cfg = {SPLIT: {"data": [{"filename": "a-1-1-0.wav"}, {"filename": "a-1-1-1.wav"}]}}
    path = os.path.join(root, "cfg.json")
    json.dump(cfg, open(path, "w"))
    with pytest.raises(ValueError, match="a-1-1-1.wav: int32"):
        WavPool(root, path, SPLIT, placement="cpu")


def test_device_placement_larger_than_free_memory_is_refused(corpus, monkeypatch):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1000, 10 ** 9))
    with pytest.raises(ValueError, match=r"\d+ bytes .* do not fit"):
        WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement="cuda")
    with pytest.raises(ValueError, match="placement must be one of"):
        WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement="hbm")


# ------------------------------------------------------------------------------ pools


def test_wav_pool_packs_int16_and_float32(corpus):
    from scipy.io import wavfile
    wavs = _pool(corpus)
    assert wavs.names == [u[0] for u in UTTS] and wavs.lens == [u[1] for u in UTTS]
    assert wavs.pcm.dtype == torch.int16 and wavs.flt.dtype == torch.float32
    assert wavs.fmt == [1 if u[2] == "f32" else 0 for u in UTTS]
    assert wavs.pcm.numel() == sum(u[1] for u in UTTS if u[2] != "f32")
    assert wavs.flt.numel() == 15000 and wavs.offs[8] == 0
    assert wavs.nbytes() == 2 * wavs.pcm.numel() + 4 * wavs.flt.numel()
    for i, (name, n, kind) in enumerate(UTTS):
        raw = wavfile.read(os.path.join(corpus["data_root"], name))[1]
        want = raw if kind == "f32" else raw.astype(np.float32) / np.float32(32768)
        assert np.array_equal(wavs.samples(i), want)


def test_wav_pool_keeps_channel_0(tmp_path):
    from scipy.io import wavfile
    root = str(tmp_path)
    x = (np.arange(400, dtype=np.int16).reshape(200, 2) * np.array([1, -1], np.int16))
    wavfile.write(os.path.join(root, "s-1-1-0.wav"), 16000, x)
    wavfile.write(os.path.join(root, "s-1-1-1.wav"), 16000, x[:, 1].copy())
    path = os.path.join(root, "cfg.json")
    json.dump({SPLIT: {"data": [{"filename": "s-1-1-0.wav"}, {"filename": "s-1-1-1.wav"}]}},
              open(path, "w"))
    wavs = WavPool(root, path, SPLIT, placement="cpu")
    assert torch.equal(wavs.pcm[:200], torch.from_numpy(x[:, 0].copy()))


def test_feature_pool_packing(corpus):
    wavs = _pool(corpus)
    fp = FeaturePool(corpus["cache"], SPLIT, "mfcc", wavs.names, "cpu")
    assert fp.F == KEYS["mfcc"] and fp.frames == [n // HOP + 1 for _, n, _ in UTTS]
    for i, name in enumerate(wavs.names):
        X = torch.load(os.path.join(corpus["cache"], SPLIT, "mfcc",
                                    os.path.splitext(name)[0] + ".mfcc"))
        got = fp.data[fp.offs[i]:fp.offs[i] + X.numel()].view(X.shape)
        assert torch.equal(got, X)
    assert fp.nbytes() == 4 * fp.data.numel()


# ------------------------------------------------------------------------------ train opts


def test_from_train_opts_on_workers_plus(corpus, tmp_path):
    root = str(tmp_path)
    data_root, cfg, cache = build_corpus(root, keys=PLUS_KEYS)
    stats = os.path.join(root, "stats.pkl")
    st = {k: {"mean": torch.arange(3075.), "std": torch.ones(3075)} for k in ("lps", "lps_long")}
    st["fbank"] = {"mean": torch.zeros(120), "std": torch.ones(120)}
    with open(stats, "wb") as fh:
        pickle.dump(st, fh)
    wavs = WavPool(data_root, cfg, SPLIT, placement="cpu")
    b = DeviceBatcher.from_train_opts(json.loads(json.dumps(WORKERS_PLUS)), T, HOP, wavs,
                                      random_scale=True, stats=stats, trans_cache=cache,
                                      feature_placement="cpu")
    assert b.mi and b.random_scale and b.d == HOP
    assert list(b.cached) == list(PLUS_KEYS)
    assert all(h == HOP and p.F == PLUS_KEYS[k] for k, (p, h) in b.cached.items())
    assert [t.name for t in b.targets] == ["lps", "lps_long"]
    lps, lpl = b.targets
    assert (lps.win, lps.n_fft, lps.hop) == (400, 2048, HOP) and lpl.win == 512
    assert torch.equal(torch.as_tensor(lps.stats[0]), st["lps"]["mean"])
    assert b.order == ["lps", "lps_long"] + list(PLUS_KEYS)
    # a target key with neither a cache nor a device implementation
    with pytest.raises(NotImplementedError, match="'fbank'"):
        DeviceBatcher.from_train_opts(WORKERS_PLUS, T, HOP, wavs, trans_cache=None)
    # single-chunk recipe: no worker named *mi*
    b = DeviceBatcher.from_train_opts({"regr": [{"name": "cchunk"}, {"name": "lps"}]}, T, HOP,
                                      wavs)
    assert not b.mi and b.cached == {} and b.targets[0].stats is None
