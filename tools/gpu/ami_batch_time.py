"""Device time of one AMI close-talk/distant-mic workers+ batch (DeviceBatcher with
dataset='ami', ihm2sdm='1,2') next to the LibriSpeech batch over the same close-talk
utterances, in one run: CUDA-event time of one plan upload + run (median over --iters batches
after warm-up) and host planner time, B=32, T=32000, with and without the PASE+ distortions
(chop / codec2 off), corpus and features in HBM.  Seeded synthetic corpus: int16 close-talk
utterances of 3 to 9 s, two distant-mic channels each (the same length, 40 samples shorter, or
1.5 to 4 s shorter, so padded tails and aliased chunks occur), fp32 features of the seven
cached workers+ keys.

Run from the repository root after build():  python tools/gpu/ami_batch_time.py [--iters 60]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from batch_time import HOP, PLUS_KEYS, measure  # noqa: E402
from distortion_banks import PASE_PLUS_P, base_cfg, build_banks  # noqa: E402
from pase_b200.batch import DeviceBatcher, FeaturePool, WavPool  # noqa: E402
from pase_b200.distortions import config_distortions  # noqa: E402
from pase_b200.targets import LPS  # noqa: E402


def corpus(root, n):
    from scipy.io import wavfile
    rng = np.random.RandomState(12)
    data_root, cache = os.path.join(root, "wavs"), os.path.join(root, "cache")
    for d in ("ihm", "sdm1", "sdm2"):
        os.makedirs(os.path.join(data_root, d))
    for k in PLUS_KEYS:
        os.makedirs(os.path.join(cache, "train", k))
    data = []
    for i in range(n):
        name = "%d-%d-%04d-%d.wav" % (100 + i // 8, 3, i // 4, i % 4)
        L = int(rng.randint(48000, 144000))
        wavfile.write(os.path.join(data_root, "ihm", name), 16000,
                      (rng.randn(L) * 3000).astype(np.int16))
        entry = {"filename": "ihm/" + name}
        for c in ("1", "2"):
            M = L - int(rng.choice([0, 40, int(rng.randint(24000, 64000))]))
            wavfile.write(os.path.join(data_root, "sdm" + c, name), 16000,
                          (rng.randn(max(M, 40000)) * 2000).astype(np.int16))
            entry[c] = "sdm%s/%s" % (c, name)
        for k, F in PLUS_KEYS.items():
            torch.save(torch.from_numpy(rng.randn(F, L // HOP + 1).astype(np.float32)),
                       os.path.join(cache, "train", k, os.path.splitext(name)[0] + "." + k))
        data.append(entry)
    cfg = os.path.join(root, "cfg.json")
    json.dump({"train": {"data": data}}, open(cfg, "w"))
    return data_root, cfg, cache


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
    B, T = 32, 32000
    with tempfile.TemporaryDirectory() as root:
        data_root, cfg, cache = corpus(root, a.utts)
        banks = build_banks(os.path.join(root, "banks"))
        dcfg = base_cfg(banks)
        dcfg.update(PASE_PLUS_P)
        dist = config_distortions(device="cuda", **dcfg)
        pools = {"librispeech": WavPool(data_root, cfg, "train", placement="cuda"),
                 "ami": WavPool(data_root, cfg, "train", placement="cuda", ihm2sdm="1,2")}
        names = pools["ami"].names
        feats = {k: (FeaturePool(cache, "train", k, names, "cuda"), HOP) for k in PLUS_KEYS}
        print("corpus: %d utterances; %.1f MB int16 close-talk audio, %.1f MB with both "
              "distant-mic channels; %.1f MB fp32 features"
              % (len(names), pools["librispeech"].nbytes() / 1e6, pools["ami"].nbytes() / 1e6,
                 sum(p.nbytes() for p, _ in feats.values()) / 1e6))
        for d, dl in ((dist, "with PASE+ distortions"), (None, "without distortions")):
            # alternate the two datasets so drifts of the shared machine hit both alike
            for rep in range(2):
                for ds in ("librispeech", "ami"):
                    b = DeviceBatcher(pools[ds], T, mi=True, random_scale=True, cached=feats,
                                      targets=[LPS(hop=HOP, name="lps"),
                                               LPS(hop=HOP, win=512, name="lps_long")],
                                      distortions=d, dataset=ds,
                                      ihm2sdm="1,2" if ds == "ami" else None)
                    med, lo, hi, host = measure(b, B, a.iters)
                    print("%-12s workers+ %-24s B=%d T=%d (pass %d): %.3f ms/batch median "
                          "(min %.3f, max %.3f) on the device (upload + kernels), host planner "
                          "%.3f ms/batch" % (ds, dl, B, T, rep, med, lo, hi, host))


if __name__ == "__main__":
    main()
