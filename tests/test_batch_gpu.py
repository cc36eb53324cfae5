"""On-device batch assembly (pase_b200/batch.py, pase_b200/csrc/batch.cu) on the GPU: the
reference's collated batches bit for bit with the corpus in HBM and in mapped page-locked host
memory, the targets and distortions against their own entry points, a B=32, T=32000 batch
against a numpy gather of the same plan, graph replay with new plans, and launch counts that
do not depend on the draws.
"""
import json
import os
import random

import numpy as np
import pytest
import torch

from batch_corpus import CASES, HOP, KEYS, SPLIT, T, digest
from distortion_banks import build_banks, case_cfg
from helpers import GOLDEN
from pase_b200 import _lib, ops
from pase_b200.batch import DeviceBatcher, FeaturePool, WavPool
from pase_b200.distortions import config_distortions
from pase_b200.targets import LPS
from test_batch import _check_batch, _seed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    from batch_corpus import build_corpus
    root = str(tmp_path_factory.mktemp("batch_corpus_gpu"))
    data_root, cfg, cache = build_corpus(root)
    banks = build_banks(os.path.join(root, "banks"))
    return dict(root=root, data_root=data_root, cfg=cfg, cache=cache, banks=banks)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "batch.pt"))


def _batcher(corpus, case, placement="cuda", targets=None):
    c = CASES[case]
    wavs = WavPool(corpus["data_root"], corpus["cfg"], SPLIT, placement=placement)
    cached = None
    if c["cached"]:
        cached = {k: (FeaturePool(corpus["cache"], SPLIT, k, wavs.names, placement), HOP)
                  for k in KEYS}
    dist = None
    if c["distortions"]:
        dist = config_distortions(device="cuda", **case_cfg("pase_plus", corpus["banks"])[0])
    return DeviceBatcher(wavs, T, mi=c["mi"], random_scale=c["random_scale"], cached=cached,
                         targets=targets, distortions=dist)


@pytest.mark.parametrize("placement", ["cuda", "pinned"])
@pytest.mark.parametrize("case", list(CASES))
def test_golden_hashes(case, placement, corpus, golden):
    meta = json.loads(golden[case + "/meta"])
    b = _batcher(corpus, case, placement)
    _seed(CASES[case]["seed"])
    for bi, idx in enumerate(CASES[case]["batches"]):
        out = b(idx)
        torch.cuda.synchronize()
        _check_batch(out, meta["arrays"][bi], case, golden.get("%s/%d/chunk" % (case, bi)))


def test_lps_and_distortions_match_their_entry_points(corpus):
    lps = LPS(hop=HOP, name="lps")
    b = _batcher(corpus, "mi_dist", targets=[lps])
    _seed(7)
    plan = b.plan([2, 6, 12, 11, 5, 10, 8, 0])
    out = b.run(b.upload(plan))
    assert torch.equal(out["lps"], LPS(hop=HOP)(out["cchunk"]))
    y, lab = b.distortions.apply(out["cchunk"], plan.dist_plan,
                                 torch.zeros_like(out["overlap"]))
    assert torch.equal(out["chunk"], y) and torch.equal(out["overlap"], lab)
    assert any(plan.samples[i]["distortions"] for i in range(plan.B))


# ---------------------------------------------------------------- B=32, T=32000 against numpy

BIG_T = 32000


def _big_corpus(root, n=48):
    from scipy.io import wavfile
    rng = np.random.RandomState(2024)
    data_root, cache = os.path.join(root, "wavs"), os.path.join(root, "cache")
    os.makedirs(os.path.join(cache, SPLIT, "prosody"))
    os.makedirs(data_root)
    data = []
    for i in range(n):
        name = "%d-%d-%04d-%d.wav" % (100 + i // 6, 7, i // 3, i % 3)
        L = int(rng.randint(BIG_T + 1, 120000)) if i % 5 else int(rng.randint(BIG_T // 2 + 1, BIG_T + 1))
        x = rng.randn(L) * 0.1
        wavfile.write(os.path.join(data_root, name), 16000,
                      x.astype(np.float32) if i % 7 == 3 else (x * 9000).astype(np.int16))
        # at least T // HOP frames, so that padded chunks have a slice too
        frames = max(L // HOP + 1, BIG_T // HOP)
        torch.save(torch.from_numpy(rng.randn(12, frames).astype(np.float32)),
                   os.path.join(cache, SPLIT, "prosody", os.path.splitext(name)[0] + ".prosody"))
        data.append({"filename": name})
    cfg = os.path.join(root, "cfg.json")
    json.dump({SPLIT: {"data": data}}, open(cfg, "w"))
    return data_root, cfg, cache


def _numpy_batch(b, plan):
    W, B = b.wavs, plan.B
    chunks = np.zeros((b.nsrc, B, 1, b.T), np.float32)
    for i, s in enumerate(plan.samples):
        for k, u in enumerate((s["index"], s["ctxt"], s["rand"])[:b.nsrc]):
            x = W.samples(u)
            L = len(x)
            p = np.arange(s["beg"][k], s["beg"][k] + b.T)
            x = x[np.where(p >= L, 2 * L - 2 - p, p)]
            if s["scale"] is not None:
                with np.errstate(invalid="ignore"):
                    x = x / np.abs(x).max() * np.float32(s["scale"][k])
            chunks[k, i, 0] = x
    feats = {}
    for key, (pool, hop) in b.cached.items():
        n = b.T // hop
        X = np.zeros((B, pool.F, n), np.float32)
        data = pool.data.cpu().numpy()
        for i, s in enumerate(plan.samples):
            u = s["index"]
            M = data[pool.offs[u]:pool.offs[u] + pool.F * pool.frames[u]].reshape(pool.F, -1)
            X[i] = M[:, s["slices"][key]:s["slices"][key] + n]
        feats[key] = X
    return chunks, feats


@pytest.mark.parametrize("placement", ["cuda", "pinned"])
def test_b32_t32000_matches_numpy_gather(placement, tmp_path):
    data_root, cfg, cache = _big_corpus(str(tmp_path))
    wavs = WavPool(data_root, cfg, SPLIT, placement=placement)
    pool = FeaturePool(cache, SPLIT, "prosody", wavs.names, placement)
    b = DeviceBatcher(wavs, BIG_T, mi=True, random_scale=True, cached={"prosody": (pool, HOP)})
    rng = np.random.RandomState(3)
    idx = [int(i) for i in rng.permutation(len(wavs))[:32]]
    g = torch.Generator()
    g.manual_seed(3)
    plan = b.plan(idx, rng=(random.Random(3), np.random.RandomState(3), g))
    assert any(wavs.lens[s["index"]] < BIG_T for s in plan.samples)      # padded chunks too
    out = b.run(b.upload(plan))
    chunks, feats = _numpy_batch(b, plan)
    for k, key in enumerate(("chunk", "chunk_ctxt", "chunk_rand")):
        assert np.array_equal(out[key].cpu().numpy(), chunks[k]), key
    assert torch.equal(out["cchunk"], out["chunk"])
    assert np.array_equal(out["prosody"].cpu().numpy(), feats["prosody"])
    assert out["overlap"].shape == (32, 1, BIG_T // HOP) and not bool(out["overlap"].any())


# ---------------------------------------------------------------- graphs and launch counts


def _full_batcher(corpus):
    return _batcher(corpus, "mi_dist", targets=[LPS(hop=HOP, name="lps"),
                                                LPS(hop=HOP, win=512, name="lps_long")])


def test_graph_replay_with_new_plans(corpus):
    b = _full_batcher(corpus)
    idx = [[2, 6, 12, 11], [5, 10, 8, 0], [1, 3, 10, 12]]
    plans = []
    for i, ix in enumerate(idx):
        b.reset()
        g = torch.Generator()
        g.manual_seed(40 + i)
        plans.append(b.plan(ix, rng=(random.Random(40 + i), np.random.RandomState(40 + i), g)))
    table = b.upload(plans[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                   # warm-up outside the capture
        b.run(table)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = b.run(table)
    for p in plans[1:]:
        b.upload(p, out=table)
        graph.replay()
        torch.cuda.synchronize()
        ref = b.run(b.upload(p))
        torch.cuda.synchronize()
        assert set(out) == set(ref)
        for k in ref:
            assert digest(out[k].cpu().numpy()) == digest(ref[k].cpu().numpy()), k


def test_launch_count_does_not_depend_on_the_draws(corpus):
    b = _full_batcher(corpus)
    b([2, 6])                                    # the first call builds the LPS constants
    counts = []
    for seed, ix in ((1, [2, 6, 12, 11]), (2, [5, 10, 8, 0]), (3, [1, 3, 10, 12])):
        b.reset()
        g = torch.Generator()
        g.manual_seed(seed)
        plan = b.plan(ix, rng=(random.Random(seed), np.random.RandomState(seed), g))
        if seed == 3:                            # no distortion drawn at all
            plan = b._pack([dict(s, distortions={}) for s in plan.samples])
        t = b.upload(plan)
        n0 = ops.launch_count
        b.run(t)
        counts.append(ops.launch_count - n0)
    torch.cuda.synchronize()
    assert counts[0] == counts[1] == counts[2], counts


def test_bad_arguments_are_refused():
    out = torch.zeros(2, 2, 100, device="cuda")
    rows = torch.zeros(2, 6, dtype=torch.int64, device="cuda")
    pcm = torch.zeros(100, dtype=torch.int16, device="cuda")
    good = [pcm, 100, None, 0, rows, 2, 1, 100, 1, out, 200]
    _lib.call("pase_chunk_gather", *good)
    for i, v, msg in [(4, None, "rows is NULL"), (9, None, "out is NULL"), (5, 0, "B="),
                      (6, 4, "nsrc"), (7, 0, "T="), (10, 199, "plane"),
                      (0, None, "both pools are NULL"), (1, -1, "pcm_len")]:
        args = list(good)
        args[i] = v
        if i == 0:
            args[1] = 0
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("pase_chunk_gather", *args)
    pool = torch.zeros(100, device="cuda")
    fr = torch.zeros(2, 3, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="pool_len"):
        _lib.call("pase_frames_gather", pool, 0, fr, 2, 4, 5, out)
    with pytest.raises(RuntimeError, match="F=0"):
        _lib.call("pase_frames_gather", pool, 100, fr, 2, 0, 5, out)
