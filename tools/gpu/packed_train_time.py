"""Cost of WaveFe.encode_packed_train's forward + backward against the zero-padded batch a
WavCollater-style loader builds (spk_id/nnet.py:70-110): the same 32 seeded utterances of 1-8 s
at 16 kHz, zero-padded to the longest and run through the uniform train encode at B=32.  PASE+
in train mode, seeded weights, per precision (3xf16 and bf16 by default), for the full sweep
(parameter gradients and dx) and the frozen one (dx only).  Host clock around work that ends in
a device synchronise; warm-up first, then the modes alternated round-robin.  Reports ms per
call and audio seconds (the real samples, not the padding) per second, and peak allocated
memory.  The card's name and power limit are read in the same run.  Prints a table, and writes
the results as JSON to --out when given.

    python tools/gpu/packed_train_time.py [--precision 3xf16 bf16] [--reps 5] [--out f.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from pase_b200 import wf_builder  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512,
             "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1}
SR = 16000


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def corpus(n=32, seed=3):
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    lens = [rng.randint(SR, 8 * SR) for _ in range(n)]
    return [(0.5 * torch.randn(T, generator=g)).cuda() for T in lens]


def run_packed(model, wavs, cots, cap):
    xs = [w.clone().requires_grad_(True) for w in wavs]
    ys = model.encode_packed_train(xs, max_samples=cap)
    sum((y * c).sum() for y, c in zip(ys, cots)).backward()


def run_padded(model, x, cot):
    x = x.clone().requires_grad_(True)
    y, _ = model.encode(x)
    (y * cot).sum().backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["3xf16", "bf16"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "packed_train_time.py needs a GPU"
    info = gpu_info()
    wavs = corpus()
    lens = [w.numel() for w in wavs]
    total, longest = sum(lens), max(lens)
    padded = torch.zeros(len(wavs), 1, longest, device="cuda")
    for i, w in enumerate(wavs):
        padded[i, 0, :w.numel()] = w
    audio_s = total / SR
    results = {"gpu": info, "utterances": len(wavs), "samples": total, "longest": longest,
               "longest_to_mean": longest * len(wavs) / total, "rows": []}
    for prec in a.precision:
        torch.manual_seed(0)
        model = wf_builder(dict(PASE_PLUS)).cuda().train()
        model.precision = prec
        with torch.no_grad():
            cots = [torch.randn_like(y) for y in model.encode_packed_train(wavs, total)]
            cot_pad = torch.randn_like(model.encode(padded)[0])
        fn = {"packed": lambda: run_packed(model, wavs, cots, total),
              "padded B=32": lambda: run_padded(model, padded, cot_pad)}
        modes = [(kind, frozen) for frozen in (False, True) for kind in fn]
        times = {m: [] for m in modes}
        peak = {}
        for rep in range(a.reps + 1):                # rep 0: warm-up
            for m in modes:
                for _, prm in model.named_parameters():   # Model.parameters(): trainable only
                    prm.requires_grad_(not m[1])
                model.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                fn[m[0]]()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if rep > 0:
                    times[m].append(dt)
                    peak[m] = max(peak.get(m, 0), torch.cuda.max_memory_allocated())
        for m in modes:
            v = sorted(times[m])
            med = v[len(v) // 2]
            results["rows"].append(dict(
                precision=prec, path=m[0], sweep="frozen (dx only)" if m[1] else "full",
                ms_median=1e3 * med, ms_min=1e3 * v[0], audio_s_per_s=audio_s / med,
                peak_alloc_gb=peak[m] / 1e9))
        del model
        torch.cuda.empty_cache()
    print("GPU:", info)
    print("%d utterances, %d samples (%.1f s of audio), longest %d, longest/mean %.2f"
          % (len(wavs), total, audio_s, longest, results["longest_to_mean"]))
    print("%-6s %-12s %-17s %10s %10s %11s %9s" % ("prec", "path", "sweep", "median ms", "min ms",
                                                   "audio s/s", "peak GB"))
    for r in results["rows"]:
        print("%-6s %-12s %-17s %10.1f %10.1f %11.0f %9.2f"
              % (r["precision"], r["path"], r["sweep"], r["ms_median"], r["ms_min"],
                 r["audio_s_per_s"], r["peak_alloc_gb"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
