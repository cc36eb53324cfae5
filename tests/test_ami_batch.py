"""On-device batch assembly of AMI close-talk/distant-mic batches (DeviceBatcher with
dataset='ami', pase_b200/batch.py), CPU side.

The pool keeps the utterances AmiSegTupleWavDataset keeps, the planner reproduces its draw
streams, the paired window takes every case of select_chunk(reuse_bounds=...), and the emulated
pipeline reproduces the reference's collated batches bit for bit (tests/golden/ami_batch.pt,
made by make_ami_batch_golden.py from the unmodified reference); reset() restores the neighbour
lists and every refusal fires before any launch.
"""
import json
import os
import random

import numpy as np
import pytest
import torch

import emul
from ami_corpus import CASES, HOP, KEYS, SPLIT, T, build_ami_corpus
from distortion_banks import build_banks, case_cfg
from helpers import GOLDEN
from make_batch_golden import BatchRecorder
from pase_b200 import ops
from pase_b200.batch import DeviceBatcher, FeaturePool, WavPool
from pase_b200.distortions import config_distortions
from test_batch import _check_batch, _normalise, _seed


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("ami_corpus"))
    data_root, cfg, cache = build_ami_corpus(root)
    banks = build_banks(os.path.join(root, "banks"))
    return dict(root=root, data_root=data_root, cfg=cfg, cache=cache, banks=banks)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ami_batch.pt"))


def ami_batcher(corpus, case, device="cpu", placement="cpu", targets=None):
    c = CASES[case]
    wavs = WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement=placement,
                   ihm2sdm=c["ihm2sdm"])
    cached = None
    if c["cached"]:
        cached = {k: (FeaturePool(corpus["cache"], SPLIT, k, wavs.names, placement), HOP)
                  for k in KEYS}
    dist = None
    if c["distortions"]:
        dist = config_distortions(device=device, **case_cfg("pase_plus", corpus["banks"])[0])
    return DeviceBatcher(wavs, T, mi=c["mi"], random_scale=c["random_scale"], cached=cached,
                         targets=targets, distortions=dist, dataset="ami", ihm2sdm=c["ihm2sdm"])


def _meta(golden, case):
    return json.loads(golden[case + "/meta"])


def _reference_log(log):
    """The reference draws the neighbour from (index, filename) pairs; the planner from the
    filenames."""
    return [["choice", ev[1], ev[2][1]] if ev[0] == "choice" and isinstance(ev[2], list) else ev
            for ev in log]


def _paired_case(b, s):
    """Which branch of select_chunk(sdm, reuse_bounds) the sample's paired window took."""
    f = b.wavs.channels[s["channel"]][s["index"]]
    L, beg = b.wavs.lens[f], s["beg"][0]
    if L <= T:
        want = "whole"
    elif beg + T <= L:
        want = "slice"
    elif beg >= L:
        return "alias"
    else:
        want = "reflect" if T - (L - beg) < L - beg else "replicate"
    assert s["paired"] == ((0 if want == "whole" else beg), want), (s["paired"], want)
    return want


# ------------------------------------------------------------------------------ pool


@pytest.mark.parametrize("case", list(CASES))
def test_pool_keeps_the_reference_utterances(case, corpus, golden):
    b = ami_batcher(corpus, case)
    assert b.wavs.names == _meta(golden, case)["names"]
    if CASES[case]["ihm2sdm"] is not None:
        assert b.wavs.dropped == ["ihm/1001-7-0002-0.wav"]
        n = len(b.wavs)
        assert sorted(b.wavs.channels) == ["1", "3"]
        for j, key in enumerate(CASES[case]["ihm2sdm"].split(",")):   # in ihm2sdm order
            files = b.wavs.channels[key]
            assert [b.wavs.files[f] for f in files] == \
                ["sdm%s/%s" % (key, x[len("ihm/"):]) for x in b.wavs.names]
            assert files == list(range((j + 1) * n, (j + 2) * n))
    else:
        assert b.wavs.channels == {} and len(b.wavs.files) == len(b.wavs)


def test_pool_reads_every_channel(corpus):
    from scipy.io import wavfile
    wavs = WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement="cpu", ihm2sdm=["1", "3"])
    assert wavs.pcm.dtype == torch.int16 and wavs.flt.dtype == torch.float32
    for i, path in enumerate(wavs.files):
        raw = wavfile.read(os.path.join(corpus["data_root"], path))[1]
        want = raw if raw.dtype == np.float32 else raw.astype(np.float32) / np.float32(32768)
        assert wavs.lens[i] == len(raw) and np.array_equal(wavs.samples(i), want), path


# ------------------------------------------------------------------------------ planner


@pytest.mark.parametrize("case", list(CASES))
def test_planner_reproduces_reference_draws(case, corpus, golden):
    meta = _meta(golden, case)
    b = ami_batcher(corpus, case)
    n = len(b.wavs)
    _seed(CASES[case]["seed"])
    k = 0
    for idx in CASES[case]["batches"]:
        for i in idx:
            with BatchRecorder() as rec:
                s = b._draw(i, random, np.random, None)
            want = meta["samples"][k]
            assert (s["index"], s["ctxt"], s["rand"], s.get("channel")) == \
                (want["index"], want["ctxt"], want["rand"], want["channel"]), (case, k)
            assert s["beg"][0] == want["chunk_beg"], (case, k)
            if want["scale"] is None:
                assert s["scale"] is None
            else:
                assert np.array_equal(np.float32(s["scale"]), np.float32(want["scale"]))
            assert _normalise(rec.log, i, n) == _reference_log(meta["logs"][k]), (case, k)
            k += 1
    assert k == len(meta["samples"])


def test_paired_windows_take_every_branch(corpus):
    seen = {}
    for case, c in CASES.items():
        if c["ihm2sdm"] is None:
            continue
        b = ami_batcher(corpus, case)
        _seed(c["seed"])
        for idx in c["batches"]:
            for s in b.plan(idx).samples:
                seen.setdefault(_paired_case(b, s), []).append(case)
    assert set(seen) == {"whole", "slice", "reflect", "replicate", "alias"}, seen
    # and in the draw-logging cases with random scales, where the alias keeps its own scale
    assert "pair_mi_scale_cached" in seen["alias"] or "pair_mi_dist" in seen["alias"], seen


def test_pool_holds_the_replicate_padding(corpus, monkeypatch):
    """Each distant-mic file shorter than its close-talk utterance by more than one sample is
    followed by copies of its last sample, as many as the longest replicate padding its paired
    window can need; a replicated window gathers F.pad(tail, mode='replicate')."""
    monkeypatch.setattr(ops, "call", emul.call)
    b = ami_batcher(corpus, "pair_mi_plain")
    W, n = b.wavs, len(b.wavs)
    for f in range(len(W.files)):
        want = max(0, W.lens[(f - n) % n] - W.lens[f] - 1) if f >= n else 0
        assert W.hold[f] == want, W.files[f]
        t = W.pcm if W.fmt[f] == 0 else W.flt
        tail = t[W.offs[f] + W.lens[f]:W.offs[f] + W.lens[f] + want]
        assert torch.equal(tail, t[W.offs[f] + W.lens[f] - 1].expand(want))
    assert W.nbytes() == 2 * W.pcm.numel() + 4 * W.flt.numel()
    # 1001-7-0001-1: close-talk 8000 samples, distant-mic 5000; beg 3500 leaves a tail of 1500
    i = W.names.index("ihm/1001-7-0001-1.wav")
    f = W.channels["1"][i]
    assert W.hold[f] == 2999 and b._paired(f, 3500) == (3500, "replicate")
    assert b._paired(f, 2500) == (2500, "reflect") and b._paired(f, 5000) is None
    for beg, mode in ((3500, "replicate"), (2500, "reflect")):
        s = dict(index=i, ctxt=i, rand=0, channel="1", files=(i, i, 0), beg=[beg, 0, 0],
                 paired=(beg, mode), scale=None, slices={})
        out = b.run(torch.from_numpy(b._pack([s]).table))
        tail = torch.from_numpy(W.samples(f)[beg:])
        want = torch.nn.functional.pad(tail.view(1, 1, -1), (0, T - len(tail)), mode=mode)
        assert torch.equal(out["chunk"].view(-1), want.view(-1)), mode
        assert torch.equal(out["cchunk"].view(-1),
                           torch.from_numpy(W.samples(i)[beg:beg + T])), mode


def test_plan_with_explicit_generators_matches_globals(corpus):
    b = ami_batcher(corpus, "pair_mi_dist")
    _seed(5)
    p1 = b.plan([3, 6, 10, 2])
    b.reset()
    g = torch.Generator()
    g.manual_seed(5)
    p2 = b.plan([3, 6, 10, 2], rng=(random.Random(5), np.random.RandomState(5), g))
    assert np.array_equal(p1.table, p2.table)
    assert p1.samples == p2.samples


def test_ihm_only_plan_is_the_librispeech_plan_without_the_zero_speech_coin(corpus):
    """Single-channel AMI over the same pool packs the same table as LibriSpeech does when the
    LibriSpeech planner's zero-speech draw is taken out of the stream."""
    ami = ami_batcher(corpus, "ihm_mi_scale_cached")
    libri = DeviceBatcher(ami.wavs, T, mi=True, random_scale=True, cached=ami.cached)

    class NoCoin:
        def __init__(self, seed):
            self.r = random.Random(seed)

        def random(self):
            return 0.5

        def choice(self, seq):
            return self.r.choice(seq)
    idx = [0, 5, 9, 3]
    pa = ami.plan(idx, rng=(random.Random(8), np.random.RandomState(8),
                            torch.Generator().manual_seed(8)))
    pl = libri.plan(idx, rng=(NoCoin(8), np.random.RandomState(8),
                              torch.Generator().manual_seed(8)))
    assert np.array_equal(pa.table, pl.table)


# ------------------------------------------------------------------------------ pipeline


@pytest.mark.parametrize("case", list(CASES))
def test_emulated_pipeline_matches_golden_hashes(case, corpus, golden, monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    meta = _meta(golden, case)
    b = ami_batcher(corpus, case)
    _seed(CASES[case]["seed"])
    for bi, idx in enumerate(CASES[case]["batches"]):
        out = b(idx)
        _check_batch(out, meta["arrays"][bi], case, golden.get("%s/%d/chunk" % (case, bi)))


def test_alias_chunk_is_the_close_talk_window(corpus, monkeypatch):
    """A distant-mic file that ends before the chunk starts: chunk is the close-talk window
    (scaled by the fourth draw), cchunk the same window (scaled by the first)."""
    monkeypatch.setattr(ops, "call", emul.call)
    b = ami_batcher(corpus, "pair_mi_plain")
    _seed(0)
    s = b._draw(2, random, np.random, None)       # IHM 20000 samples, SDMs of 4400 / 4500
    s = dict(s, beg=[9000] + s["beg"][1:], paired=b._paired(
        b.wavs.channels[s["channel"]][2], 9000), scale=[0.25, 0.5, 0.75, 0.125], slices={})
    assert s["paired"] is None
    b.random_scale = True
    out = b.run(torch.from_numpy(b._pack([s]).table))
    x = torch.from_numpy(b.wavs.samples(2)[9000:9000 + T])
    m = x.abs().max()
    assert torch.equal(out["chunk"].view(-1), x / m * torch.tensor(0.125))
    assert torch.equal(out["cchunk"].view(-1), x / m * torch.tensor(0.25))


# ------------------------------------------------------------------------------ reset


def test_neighbour_lists_shrink_and_reset_restores_them(corpus):
    b = ami_batcher(corpus, "pair_mi_plain")
    full = {k: list(v) for k, v in b._neighbors.items()}
    _seed(1)
    b.plan([0, 1, 2])
    assert b._neighbors["ihm/1001-7-0001-"] == ["ihm/1001-7-0001-3.wav"]
    with BatchRecorder() as rec:
        s = b._draw(3, random, np.random, None)
    assert s["ctxt"] == 3                      # empty list: the utterance's own SDM, no draw
    assert rec.log[0][:2] == ["choice", len(b.wavs) - 1]
    with pytest.raises(ValueError, match="visited twice"):
        b.plan([2])
    b.reset()
    assert b._neighbors == full


# ------------------------------------------------------------------------------ refusals


def _counting(monkeypatch):
    calls = []
    monkeypatch.setattr(ops, "call", lambda name, *a: calls.append(name))
    return calls


def test_refusals_fire_before_any_launch(corpus, tmp_path, monkeypatch):
    calls = _counting(monkeypatch)
    root, cfg = corpus["data_root"], corpus["cfg"]
    wavs = WavPool(root, cfg, SPLIT, placement="cpu", ihm2sdm="1,3")
    with pytest.raises(ValueError, match="zero_speech_p=0.1 must be 0"):
        DeviceBatcher(wavs, T, dataset="ami", ihm2sdm="1,3", zero_speech_p=0.1)
    with pytest.raises(ValueError, match="channel key '2' of ihm2sdm=1,2 is in no entry"):
        WavPool(root, cfg, SPLIT, placement="cpu", ihm2sdm="1,2")
    with pytest.raises(ValueError, match="ihm2sdm=\\['3'\\], the pool was loaded with"):
        DeviceBatcher(wavs, T, dataset="ami", ihm2sdm=["3"])
    with pytest.raises(ValueError, match="'ami' dataset only"):
        DeviceBatcher(wavs, T)
    with pytest.raises(ValueError, match="'PairWavDataset' is not assembled"):
        DeviceBatcher(wavs, T, dataset="PairWavDataset", ihm2sdm="1,3")
    # a distant-mic file of at most T samples that F.pad cannot reflect-pad to T: the SDM of
    # 5005-4-0007-1 on channel 1 has 3600 samples, so T = 7300 leaves padding 3700 >= 3600
    b = DeviceBatcher(wavs, 7300, mi=False, dataset="ami", ihm2sdm="1,3")
    i = wavs.names.index("ihm/5005-4-0007-1.wav")

    class Channel1(random.Random):
        def choice(self, seq):
            return "1" if seq == ["1", "3"] else super().choice(seq)
    with pytest.raises(ValueError, match="distant-mic file sdm1/5005-4-0007-1.wav: 3600 samples"):
        b.plan([i], rng=(Channel1(0), np.random.RandomState(0), torch.Generator()))
    # the context / random windows on a short SDM refuse as the IHM windows do
    b = DeviceBatcher(wavs, 7300, mi=True, dataset="ami", ihm2sdm="1,3")
    with pytest.raises(ValueError, match="cannot be reflect-padded"):
        for s in range(20):
            b.reset()
            b.plan(list(range(len(wavs))), rng=(random.Random(s), np.random.RandomState(s),
                                                torch.Generator().manual_seed(s)))
    assert calls == []


def test_from_train_opts_takes_the_dataset_options(corpus):
    wavs = WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement="cpu", ihm2sdm="1,3")
    wcfg = {"regr": [{"name": "cchunk"}, {"name": "fbank"}], "cls": [{"name": "mi"}]}
    b = DeviceBatcher.from_train_opts(wcfg, T, HOP, wavs, random_scale=True,
                                      trans_cache=corpus["cache"], feature_placement="cpu",
                                      dataset=["AmiSegTupleWavDataset"], ihm2sdm="1,3")
    assert (b.dataset, b.ihm2sdm, b.paired, b.mi) == ("ami", ["1", "3"], True, True)
    assert b.cached["fbank"][0].frames[0] == 9000 // HOP + 1         # the IHM utterance's
    with pytest.raises(ValueError, match="'GenhancementDataset' is not assembled"):
        DeviceBatcher.from_train_opts(wcfg, T, HOP, wavs, trans_cache=corpus["cache"],
                                      feature_placement="cpu", dataset="GenhancementDataset")
    with pytest.raises(NotImplementedError, match="MetaWavConcatDataset"):
        DeviceBatcher.from_train_opts(wcfg, T, HOP, wavs, trans_cache=corpus["cache"],
                                      feature_placement="cpu",
                                      dataset=["AmiSegTupleWavDataset"] * 2, ihm2sdm="1,3")
    single = WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement="cpu")
    b = DeviceBatcher.from_train_opts(wcfg, T, HOP, single, trans_cache=corpus["cache"],
                                      feature_placement="cpu", dataset="AmiSegTupleWavDataset")
    assert (b.dataset, b.paired, len(b.wavs)) == ("ami", False, 12)
