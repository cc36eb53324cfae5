"""Feature extraction throughput of PASE+ (eval) over a seeded TIMIT-like corpus: ~1000
utterances, lengths uniform over 1-8 s at 16 kHz, in 3xf16 and bf16.
  (a) the reference's downstream loop: one B=1 ``model(x, mode='avg_norm')`` per utterance
      (ASR/run_TIMIT_fast.py:119-127), CPU waveform moved to the GPU per call;
  (b) ``model.extract(wavs, mode='avg_norm')`` (packed variable-length forwards).
Both warm up first, are timed with a host clock around work that ends in a device
synchronise, and their outputs are compared for equality in the same run.  Reports
audio-seconds per second of (a) and (b) and their ratio, with the card name and power limit.
Run from the repository root after build():
    python tools/gpu/extract_time.py [--n 1000] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from detweights import fill_state_dict  # noqa: E402
from helpers import resolve_cfg  # noqa: E402
from pase_b200.frontend import WaveFe  # noqa: E402

SR = 16000


def corpus(n, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1 * SR, 8 * SR + 1, size=n)
    return [torch.from_numpy(rng.standard_normal(int(T)).astype(np.float32) * 0.5)
            for T in lengths]


def timed(fn, reps):
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        q = torch.cuda.get_device_name()
    print("device:", q)
    wavs = corpus(a.n, a.seed)
    audio_s = sum(w.numel() for w in wavs) / SR
    print("corpus: %d utterances, %.1f s of audio" % (len(wavs), audio_s))
    for prec in ("3xf16", "bf16"):
        m = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg"))
        m.load_state_dict(fill_state_dict(m.state_dict(), 11))
        m.precision = prec
        m = m.cuda().eval()

        def loop():
            with torch.no_grad():
                return [m(w.view(1, 1, -1).cuda(), mode="avg_norm") for w in wavs]

        def packed():
            return m.extract(wavs, mode="avg_norm")

        loop()                                  # warm-up: every B=1 plan shape, modules
        packed()
        t_loop, out_loop = timed(loop, a.reps)
        t_pack, out_pack = timed(packed, a.reps)
        equal = sum(torch.equal(x, y) for x, y in zip(out_loop, out_pack))
        maxdiff = max(float((x - y).abs().max()) for x, y in zip(out_loop, out_pack))
        row = dict(precision=prec, utterances=len(wavs), audio_s=round(audio_s, 1),
                   loop_s=round(t_loop, 4), extract_s=round(t_pack, 4),
                   loop_audio_s_per_s=round(audio_s / t_loop, 1),
                   extract_audio_s_per_s=round(audio_s / t_pack, 1),
                   ratio=round(t_loop / t_pack, 2), bit_equal=equal, max_abs_diff=maxdiff,
                   plan_bytes=[p.nbytes() for p in m._packed_plans.values()],
                   device=q)
        print(json.dumps(row))
        del out_loop, out_pack


if __name__ == "__main__":
    main()
