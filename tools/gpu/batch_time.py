"""Time per batch of the on-device batch assembly (pase_b200/batch.py): CUDA-event time of one
plan upload + run (median over --iters batches after warm-up) and host planner time, on a seeded
synthetic corpus (int16 utterances of 3 to 9 s, fp32 features of the seven cached workers+ keys,
synthetic distortion banks of tests/golden/distortion_banks.py).  Configurations:

  workers+       B=32, T=32000: lps / lps_long on the device, seven cached keys, PASE+
                 distortions (chop / codec2 off); features in HBM, then in pinned host memory
  gather only    the same batch without targets and distortions (the batch.cu kernels + upload)
  config 5       B=64, T=48000, workers+ recipe, features in HBM

Run from the repository root after build():  python tools/gpu/batch_time.py [--iters 60]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from distortion_banks import PASE_PLUS_P, base_cfg, build_banks  # noqa: E402
from pase_b200.batch import DeviceBatcher, FeaturePool, WavPool  # noqa: E402
from pase_b200.distortions import config_distortions  # noqa: E402
from pase_b200.targets import LPS  # noqa: E402

HOP = 160
PLUS_KEYS = {"fbank": 120, "fbank_long": 120, "gtn": 120, "gtn_long": 120, "mfcc": 39,
             "mfcc_long": 60, "prosody": 12}


def corpus(root, n):
    from scipy.io import wavfile
    rng = np.random.RandomState(11)
    data_root, cache = os.path.join(root, "wavs"), os.path.join(root, "cache")
    os.makedirs(data_root)
    for k in PLUS_KEYS:
        os.makedirs(os.path.join(cache, "train", k))
    data = []
    for i in range(n):
        name = "%d-%d-%04d-%d.wav" % (100 + i // 8, 3, i // 4, i % 4)
        L = int(rng.randint(48000, 144000))
        wavfile.write(os.path.join(data_root, name), 16000,
                      (rng.randn(L) * 3000).astype(np.int16))
        for k, F in PLUS_KEYS.items():
            torch.save(torch.from_numpy(rng.randn(F, L // HOP + 1).astype(np.float32)),
                       os.path.join(cache, "train", k, os.path.splitext(name)[0] + "." + k))
        data.append({"filename": name})
    cfg = os.path.join(root, "cfg.json")
    json.dump({"train": {"data": data}}, open(cfg, "w"))
    return data_root, cfg, cache


def plans(b, B, count):
    """`count` plans drawn epoch by epoch from shuffled indices (reset() per epoch)."""
    n = len(b.wavs)
    out, host = [], []
    while len(out) < count:
        b.reset()
        perm = np.random.permutation(n)
        for j in range(0, n - B + 1, B):
            t0 = time.perf_counter()
            out.append(b.plan(perm[j:j + B].tolist()))
            host.append((time.perf_counter() - t0) * 1e3)
    return out[:count], statistics.median(host)


def measure(b, B, iters, warm=5):
    ps, host_ms = plans(b, B, iters + warm)
    for p in ps[:warm]:
        b.run(b.upload(p))
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
           for _ in range(iters)]
    for p, (e0, e1) in zip(ps[warm:], evs):
        e0.record()
        b.run(b.upload(p))
        e1.record()
    torch.cuda.synchronize()
    ms = [e0.elapsed_time(e1) for e0, e1 in evs]
    return statistics.median(ms), min(ms), max(ms), host_ms


def algorithmic_mb(b, B, T):
    """HBM bytes the batch.cu kernels need: pool reads once, every output written once."""
    src = 2 if b.wavs.pcm is not None else 4
    chunks = B * b.nsrc * T * src + (b.nsrc + 1) * B * T * 4
    feats = sum(2 * B * p.F * (T // h) * 4 for p, h in b.cached.values())
    return chunks / 1e6, feats / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--utts", type=int, default=160)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device:", q or torch.cuda.get_device_name())
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    with tempfile.TemporaryDirectory() as root:
        data_root, cfg, cache = corpus(root, a.utts)
        banks = build_banks(os.path.join(root, "banks"))
        dcfg = base_cfg(banks)
        dcfg.update(PASE_PLUS_P)
        dist = config_distortions(device="cuda", **dcfg)
        wavs = WavPool(data_root, cfg, "train", placement="cuda")
        feats = {pl: {k: (FeaturePool(cache, "train", k, wavs.names, pl), HOP) for k in PLUS_KEYS}
                 for pl in ("cuda", "pinned")}
        print("corpus: %d utterances, %.1f MB int16 audio, %.1f MB fp32 features"
              % (len(wavs), wavs.nbytes() / 1e6,
                 sum(p.nbytes() for p, _ in feats["cuda"].values()) / 1e6))

        def targets():
            return [LPS(hop=HOP, name="lps"), LPS(hop=HOP, win=512, name="lps_long")]
        runs = [("workers+, features in HBM", 32, 32000, feats["cuda"], targets(), dist),
                ("workers+, features pinned", 32, 32000, feats["pinned"], targets(), dist),
                ("gather only, HBM", 32, 32000, feats["cuda"], [], None),
                ("gather only, pinned", 32, 32000, feats["pinned"], [], None),
                ("config 5 (workers+), HBM", 64, 48000, feats["cuda"], targets(), dist)]
        for label, B, T, cached, tg, d in runs:
            b = DeviceBatcher(wavs, T, mi=True, random_scale=True, cached=cached, targets=tg,
                              distortions=d)
            med, lo, hi, host = measure(b, B, a.iters)
            mb_c, mb_f = algorithmic_mb(b, B, T)
            print("%-28s B=%d T=%d: %.3f ms/batch median (min %.3f, max %.3f) on the device "
                  "(upload + kernels), host planner %.3f ms/batch; batch.cu algorithmic bytes "
                  "%.1f MB chunks + %.1f MB cached targets"
                  % (label, B, T, med, lo, hi, host, mb_c, mb_f))


if __name__ == "__main__":
    main()
