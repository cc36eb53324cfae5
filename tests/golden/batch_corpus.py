"""Deterministic synthetic corpus for the batch-assembly goldens (tests/golden/batch.pt):
LibriSpeech-style names <spk>-<chap>-<utt>-<seg>.wav in prefix groups of 1 to 4 segments,
lengths below, equal to, one above and far above the chunk size, one float32 wav, one silent
utterance, cached fp32 features for two keys (the torch.save layout of precompute_aco_data.py)
and a data_cfg json.  make_batch_golden.py and the tests rebuild the same files from these
seeds, so no audio is committed.
"""
import json
import os

import numpy as np
import torch

T = 4000                     # chunk size of the golden cases
HOP = 160
SPLIT = "train"
KEYS = {"fbank": 6, "mfcc": 4}          # cached key -> F

# (name, length, kind): kind 'pcm' (int16), 'f32' (float32 wav) or 'zero' (silent int16)
UTTS = [
    ("1001-134707-0001-0.wav", 9000, "pcm"),
    ("1001-134707-0001-1.wav", 4000, "pcm"),     # = T
    ("1001-134707-0001-2.wav", 37000, "pcm"),
    ("1001-134707-0001-3.wav", 4001, "pcm"),     # = T + 1
    ("1001-134707-0002-0.wav", 2500, "pcm"),     # < T: reflect padded
    ("1001-134707-0002-1.wav", 12000, "pcm"),
    ("1001-134707-0002-2.wav", 20000, "pcm"),
    ("2002-7-0005-0.wav", 3100, "pcm"),          # < T
    ("2002-7-0005-1.wav", 15000, "f32"),
    ("3003-9-0010-0.wav", 6000, "zero"),         # silent: norm_and_scale gives NaN
    ("4004-2-0003-0.wav", 8000, "pcm"),
    ("4004-2-0003-1.wav", 26000, "pcm"),
    ("5005-4-0007-0.wav", 11000, "pcm"),
]


def make_samples(i, n, kind):
    rng = np.random.RandomState(1000 + i)
    if kind == "zero":
        return np.zeros(n, dtype=np.int16)
    env = 0.3 + 0.7 * np.abs(np.sin(np.linspace(0, 3.0 + i, n)))
    x = rng.randn(n) * env
    if kind == "f32":
        return (0.2 * x).astype(np.float32)
    return np.clip(x * 3000, -32768, 32767).astype(np.int16)


def frame_count(n):
    """Frames of a feature computed over a whole utterance of n samples (centred frames)."""
    return n // HOP + 1


def make_features(i, key, F, n):
    rng = np.random.RandomState(5000 + 17 * i + len(key))
    return torch.from_numpy(rng.randn(F, frame_count(n)).astype(np.float32))


def build_corpus(root, keys=KEYS):
    """Writes the corpus under `root`, with cached features for `keys` ({key: F}); returns
    (data_root, data_cfg path, trans_cache)."""
    from scipy.io import wavfile
    data_root = os.path.join(root, "wavs")
    cache = os.path.join(root, "cache")
    os.makedirs(data_root, exist_ok=True)
    for i, (name, n, kind) in enumerate(UTTS):
        wavfile.write(os.path.join(data_root, name), 16000, make_samples(i, n, kind))
        base = os.path.splitext(name)[0]
        for key, F in keys.items():
            d = os.path.join(cache, SPLIT, key)
            os.makedirs(d, exist_ok=True)
            torch.save(make_features(i, key, F, n), os.path.join(d, base + "." + key))
    spks = sorted({u[0].split("-")[0] for u in UTTS})
    cfg = {"speakers": spks,
           SPLIT: {"data": [{"filename": u[0], "speaker": u[0].split("-")[0]} for u in UTTS],
                   "speakers": spks, "total_wav_dur": sum(u[1] for u in UTTS)}}
    cfg_path = os.path.join(root, "data_cfg.json")
    with open(cfg_path, "w") as fh:
        json.dump(cfg, fh)
    return data_root, cfg_path, cache


# name -> dict(mi, random_scale, cached, distortions, seed, batches)
# Cached keys only with chunks of >= T samples: a padded chunk has fewer frames than T // HOP.
CASES = {
    "mi_scale_cached": dict(mi=True, random_scale=True, cached=True, distortions=False, seed=31,
                            batches=[[0, 2, 5, 6, 11, 12], [1, 3, 10, 8, 9]]),
    "single_short": dict(mi=False, random_scale=True, cached=False, distortions=False, seed=32,
                         batches=[[4, 1, 3, 7, 9, 8, 12]]),
    "mi_short": dict(mi=True, random_scale=False, cached=False, distortions=False, seed=33,
                     batches=[[4, 7, 1, 3, 9, 8, 5, 2]]),
    "mi_dist": dict(mi=True, random_scale=True, cached=True, distortions=True, seed=34,
                    batches=[[2, 6, 12, 11, 5, 10, 8, 0]]),
}


def digest(x):
    """SHA-256 of a float32 array's shape and bytes, NaNs made canonical (CPU and GPU NaN
    payloads differ; the comparison is otherwise bit for bit)."""
    import hashlib
    a = np.array(x, dtype=np.float32, order="C", copy=True)
    nan = np.isnan(a)
    bits = a.view(np.uint32)
    bits[nan] = 0x7FC00000
    h = hashlib.sha256(repr(tuple(a.shape)).encode())
    h.update(bits.tobytes())
    return h.hexdigest()
