"""Cost of WaveFe.encode_packed's forward + backward against a B=1 encode + backward loop over the
same utterances (PASE+ in eval mode, seeded weights, a seeded corpus of 1-8 s utterances at
16 kHz grouped into full packs of EXTRACT_MAX_SAMPLES samples), per precision (3xf16 and bf16
by default), for the full sweep (parameter gradients and dx) and the frozen one (dx only).
Host clock around work that ends in a device synchronise; warm-up first, then the modes
alternated round-robin.  Peak allocated memory per mode.  The card's name and power limit are
read in the same run.  Prints a table, and writes the results as JSON to --out when given.

    python tools/gpu/packed_grad_time.py [--precision 3xf16 bf16] [--reps 5] [--out f.json]
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
from pase_b200.frontend import EXTRACT_MAX_SAMPLES  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512,
             "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def corpus(npacks, seed=3):
    """Packs of 1-8 s utterances, each filled up to EXTRACT_MAX_SAMPLES."""
    rng = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    packs = []
    for _ in range(npacks):
        lens, total = [], 0
        while True:
            T = rng.randint(16000, 128000)
            if total + T > EXTRACT_MAX_SAMPLES:
                break
            lens.append(T)
            total += T
        packs.append([(0.5 * torch.randn(T, generator=g)).cuda() for T in lens])
    return packs


def set_frozen(model, frozen):
    for _, p in model.named_parameters():
        p.requires_grad_(not frozen)


def run_packed(model, pack, cots):
    xs = [w.clone().requires_grad_(True) for w in pack]
    ys = model.encode_packed(xs)
    sum((y * c).sum() for y, c in zip(ys, cots)).backward()


def run_loop(model, pack, cots):
    for w, c in zip(pack, cots):
        x = w.view(1, 1, -1).clone().requires_grad_(True)
        y, _ = model.encode(x)
        (y * c).sum().backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["3xf16", "bf16"])
    ap.add_argument("--packs", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "packed_grad_time.py needs a GPU"
    info = gpu_info()
    packs = corpus(a.packs)
    results = {"gpu": info, "packs": a.packs, "utterances": sum(len(p) for p in packs),
               "samples": sum(w.numel() for p in packs for w in p), "rows": []}
    for prec in a.precision:
        torch.manual_seed(0)
        model = wf_builder(dict(PASE_PLUS)).cuda().eval()
        model.precision = prec
        model.MAX_PLANS = 64             # the B=1 loop holds one plan per length
        with torch.no_grad():
            cots = [[torch.randn_like(y) for y in model.extract(p)] for p in packs]
        modes = [(kind, frozen) for frozen in (False, True) for kind in ("packed", "loop")]
        fn = {"packed": run_packed, "loop": run_loop}
        times = {m: [] for m in modes}
        peak = {}
        for rep in range(a.reps + 1):                # rep 0: warm-up
            for m in modes:
                set_frozen(model, m[1])
                model.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                for p, c in zip(packs, cots):
                    fn[m[0]](model, p, c)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if rep > 0:
                    times[m].append(dt)
                    peak[m] = max(peak.get(m, 0), torch.cuda.max_memory_allocated())
        for m in modes:
            v = sorted(times[m])
            row = dict(precision=prec, path=m[0], sweep="frozen (dx only)" if m[1] else "full",
                       ms_median=1e3 * v[len(v) // 2], ms_min=1e3 * v[0],
                       peak_alloc_gb=peak[m] / 1e9)
            results["rows"].append(row)
        del model
        torch.cuda.empty_cache()
    print("GPU:", info)
    print("%d packs, %d utterances, %d samples" % (a.packs, results["utterances"],
                                                   results["samples"]))
    print("%-6s %-7s %-17s %10s %10s %9s" % ("prec", "path", "sweep", "median ms", "min ms",
                                              "peak GB"))
    for r in results["rows"]:
        print("%-6s %-7s %-17s %10.1f %10.1f %9.2f" % (r["precision"], r["path"], r["sweep"],
                                                      r["ms_median"], r["ms_min"],
                                                      r["peak_alloc_gb"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
