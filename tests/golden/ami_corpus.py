"""Deterministic synthetic paired corpus for the AMI batch-assembly goldens
(tests/golden/ami_batch.pt): close-talk (IHM) wavs under ihm/ with distant-mic (SDM) wavs of
channels '1' and '3' under sdm1/ and sdm3/, named <spk>-<chap>-<utt>-<seg>.wav in prefix
groups of 1 to 4 segments.  The SDM lengths put the paired window (the IHM chunk's bounds on
the SDM) in every case of select_chunk(reuse_bounds=...): shorter than T (the whole file,
reflect-padded), the plain slice, a tail padded by reflect or by replicate, and a chunk start
past the SDM's end.  One entry lacks channel '3', one IHM wav is silent, some wavs are
float32.  Cached fp32 features exist for the IHM utterances only.  make_ami_batch_golden.py
and the tests rebuild the same files from these seeds, so no audio is committed.
"""
import json
import os

import numpy as np
import torch

from batch_corpus import HOP, KEYS, SPLIT, T, digest, make_features, make_samples  # noqa: F401

CHANNELS = ("1", "3")
# (IHM name, IHM length, IHM kind, {channel: (SDM length, SDM kind)})
ENTRIES = [
    ("1001-7-0001-0.wav", 9000, "pcm", {"1": (9000, "pcm"), "3": (9005, "pcm")}),
    ("1001-7-0001-1.wav", 8000, "pcm", {"1": (5000, "pcm"), "3": (5000, "f32")}),
    ("1001-7-0001-2.wav", 20000, "pcm", {"1": (4500, "pcm"), "3": (4400, "pcm")}),
    ("1001-7-0001-3.wav", 3950, "pcm", {"1": (3000, "pcm"), "3": (4100, "pcm")}),
    ("1001-7-0002-0.wav", 12000, "pcm", {"1": (12000, "pcm")}),            # lacks '3'
    ("1001-7-0002-1.wav", 8000, "f32", {"1": (6000, "pcm"), "3": (6000, "f32")}),
    ("2002-4-0005-0.wav", 15000, "pcm", {"1": (7100, "pcm"), "3": (7000, "pcm")}),
    ("3003-9-0010-0.wav", 6000, "pcm", {"1": (6000, "pcm"), "3": (5990, "pcm")}),
    ("3003-9-0010-1.wav", 26000, "pcm", {"1": (25000, "pcm"), "3": (26000, "f32")}),
    ("4004-2-0003-0.wav", 11000, "zero", {"1": (11000, "pcm"), "3": (10000, "pcm")}),
    ("5005-4-0007-0.wav", 9500, "pcm", {"1": (4700, "pcm"), "3": (9500, "f32")}),
    ("5005-4-0007-1.wav", 7000, "pcm", {"1": (3600, "pcm"), "3": (3900, "pcm")}),
]


def sdm_name(ch, name):
    return "sdm%s/%s" % (ch, name)


def build_ami_corpus(root, keys=KEYS):
    """Writes the corpus under `root`; returns (data_root, data_cfg path, trans_cache)."""
    from scipy.io import wavfile
    data_root, cache = os.path.join(root, "wavs"), os.path.join(root, "cache")
    for d in ["ihm"] + ["sdm" + c for c in CHANNELS]:
        os.makedirs(os.path.join(data_root, d), exist_ok=True)
    data = []
    for i, (name, n, kind, sdms) in enumerate(ENTRIES):
        wavfile.write(os.path.join(data_root, "ihm", name), 16000, make_samples(i, n, kind))
        entry = {"filename": "ihm/" + name, "speaker": name.split("-")[0]}
        for c, (m, k) in sdms.items():
            x = make_samples(100 * (1 + int(c)) + i, m, k)
            wavfile.write(os.path.join(data_root, sdm_name(c, name)), 16000, x)
            entry[c] = sdm_name(c, name)
        data.append(entry)
        for key, F in keys.items():
            d = os.path.join(cache, SPLIT, key)
            os.makedirs(d, exist_ok=True)
            torch.save(make_features(i, key, F, n),
                       os.path.join(d, os.path.splitext(name)[0] + "." + key))
    spks = sorted({e[0].split("-")[0] for e in ENTRIES})
    cfg = {"speakers": spks,
           SPLIT: {"data": data, "speakers": spks, "total_wav_dur": sum(e[1] for e in ENTRIES)}}
    cfg_path = os.path.join(root, "ami_cfg.json")
    with open(cfg_path, "w") as fh:
        json.dump(cfg, fh)
    return data_root, cfg_path, cache


# name -> dict(mi, random_scale, cached, distortions, ihm2sdm, seed, batches); with ihm2sdm
# the pool holds 11 utterances (entry 4 is dropped), without it 12.
CASES = {
    "pair_mi_scale_cached": dict(mi=True, random_scale=True, cached=True, distortions=False,
                                 ihm2sdm="1,3", seed=41,
                                 batches=[[0, 2, 5, 6, 9, 10], [1, 3, 4, 8, 7]]),
    "pair_mi_plain": dict(mi=True, random_scale=False, cached=False, distortions=False,
                          ihm2sdm="1,3", seed=42,
                          batches=[[3, 7, 1, 10, 9, 8], [0, 5, 4, 2, 6]]),
    "pair_single_scale": dict(mi=False, random_scale=True, cached=False, distortions=False,
                              ihm2sdm="3,1", seed=43,
                              batches=[[6, 2, 9, 0, 4, 1, 10, 8, 3, 5, 7]]),
    "pair_mi_dist": dict(mi=True, random_scale=True, cached=True, distortions=True,
                         ihm2sdm="1,3", seed=44,
                         batches=[[2, 6, 10, 4, 5, 8, 0, 9], [1, 3, 7]]),
    "ihm_mi_scale_cached": dict(mi=True, random_scale=True, cached=True, distortions=False,
                                ihm2sdm=None, seed=45,
                                batches=[[0, 2, 5, 6, 11, 9], [1, 3, 10, 8, 7, 4]]),
}
