"""Generates tests/golden/batch.pt from the UNMODIFIED reference data pipeline
(pase/dataset.py LibriSpeechSegTupleWavDataset + DictCollater, pase/transforms.py
CachedCompose + MIChunkWav / SingleChunkWav, and config_distortions for the distorted case).
Run:
    PASE_REFERENCE_ROOT=<checkout of santi-pdp/pase> python tests/golden/make_batch_golden.py

Import stubs as make_distortion_golden.py, plus torchaudio.load on scipy's wav reader (PCM16 as
k / 32768 in float32, float32 as is, (channels, frames) as torchaudio returns).  For each case
the corpus of batch_corpus.py is built, the global random / np.random / torch generators are
seeded once, and the dataset's __getitem__ runs on each index of each batch in turn (what a
num_workers=0 DataLoader does), then DictCollater collates.  Kept per case: every draw of every
sample (random.random, random.choice, np.random.randint, torch.rand), the parsed per-sample
choices, and per batch the shape and SHA-256 (batch_corpus.digest) of every clean collated
array, the first values of each, and for the distorted case the distorted chunk itself.
"""
import json
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from batch_corpus import CASES, HOP, KEYS, SPLIT, T, UTTS, build_corpus, digest  # noqa: E402
from distortion_banks import build_banks, case_cfg  # noqa: E402
from make_distortion_golden import Recorder, install_stubs  # noqa: E402

REF_ROOT = os.environ.get("PASE_REFERENCE_ROOT", "")
VIEW = 8


class BatchRecorder(Recorder):
    """Recorder that also logs torch.rand(1) draws (norm_and_scale)."""

    def __enter__(self):
        super().__enter__()
        self._rand = torch.rand
        r0 = self._rand

        def rand(*a, **k):
            v = r0(*a, **k)
            self.log.append(["rand", float(v.reshape(-1)[0])])
            return v
        torch.rand = rand
        return self

    def __exit__(self, *exc):
        torch.rand = self._rand
        super().__exit__(*exc)


def install_torchaudio_stub():
    from scipy.io import wavfile

    def load(path):
        rate, data = wavfile.read(path)
        if data.dtype == np.int16:
            x = data.astype(np.float32) / np.float32(32768.0)
        else:
            assert data.dtype == np.float32, data.dtype
            x = data
        x = x.reshape(len(x), -1).T
        return torch.from_numpy(np.ascontiguousarray(x)), rate
    m = types.ModuleType("torchaudio")
    m.load = load
    sys.modules["torchaudio"] = m


def parse(index, log, mi, n):
    """Per-sample choices from the draw log of one __getitem__."""
    names = [u[0] for u in UTTS]
    lens = [u[1] for u in UTTS]
    assert log[0][0] == "random"
    k = 1
    if log[1][0] == "choice" and log[2][0] == "choice":
        ctxt = names.index(log[1][2])
        k = 2
    else:
        ctxt = index
    assert log[k][0] == "choice" and log[k][1] == n - 1
    rand = int(log[k][2])
    k += 1
    srcs = (index, ctxt, rand) if mi else (index,)
    beg = []
    for i in srcs:
        if lens[i] > T:
            assert log[k][0] == "randint" and log[k][1:3] == [0, lens[i] - T]
            beg.append(log[k][3])
            k += 1
        else:
            beg.append(0)
    scale = []
    while k < len(log) and log[k][0] == "rand":
        scale.append(log[k][1])
        k += 1
    return {"index": index, "ctxt": ctxt, "rand": rand, "beg": beg,
            "scale": scale or None, "dist_log": log[k:]}


def main():
    if not os.path.isdir(os.path.join(REF_ROOT, "pase")):
        raise SystemExit("set PASE_REFERENCE_ROOT to a checkout of santi-pdp/pase")
    install_stubs()
    install_torchaudio_stub()
    sys.path.insert(0, REF_ROOT)
    import pase.transforms as RT
    from pase.dataset import DictCollater, LibriSpeechSegTupleWavDataset
    out = {}
    with tempfile.TemporaryDirectory() as root:
        data_root, cfg_path, cache = build_corpus(root)
        bank_paths = build_banks(os.path.join(root, "banks"))
        for name, c in CASES.items():
            chunker = (RT.MIChunkWav if c["mi"] else RT.SingleChunkWav)(
                T, random_scale=c["random_scale"])
            trans, keys = [RT.ToTensor(), chunker], ["totensor", "chunk"]
            if c["cached"]:
                trans += [RT.FBanks(hop=HOP, name="fbank"), RT.MFCC(hop=HOP, name="mfcc")]
                keys += list(KEYS)
            dist = None
            if c["distortions"]:
                dist = RT.config_distortions(**case_cfg("pase_plus", bank_paths)[0])
            ds = LibriSpeechSegTupleWavDataset(
                data_root, cfg_path, SPLIT, transform=RT.CachedCompose(trans, keys, cache),
                distortion_transforms=dist, zero_speech_p=0)
            coll = DictCollater()
            random.seed(c["seed"])
            np.random.seed(c["seed"])
            torch.manual_seed(c["seed"])
            meta = {"samples": [], "logs": [], "arrays": []}
            for bi, idx in enumerate(c["batches"]):
                pkgs = []
                for i in idx:
                    with BatchRecorder() as rec:
                        pkgs.append(ds[i])
                    meta["logs"].append(rec.log)
                    meta["samples"].append(parse(i, rec.log, c["mi"], len(UTTS)))
                    assert pkgs[-1]["chunk_beg_i"] == meta["samples"][-1]["beg"][0]
                batch = coll(pkgs)
                arr = {}
                for k, v in batch.items():
                    a = v.float().numpy()
                    if c["distortions"] and k == "chunk":
                        out["%s/%d/chunk" % (name, bi)] = v.float().clone()
                        continue
                    arr[k] = {"shape": list(a.shape), "sha256": digest(a),
                              "view": [float(x) for x in a.reshape(a.shape[0], -1)[0, :VIEW]]}
                meta["arrays"].append(arr)
            out[name + "/meta"] = json.dumps(meta)
            print("%-16s %s" % (name, {k: v["shape"] for k, v in meta["arrays"][0].items()}))
    torch.save(out, os.path.join(HERE, "batch.pt"))


if __name__ == "__main__":
    main()
