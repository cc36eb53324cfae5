"""Cost of WaveFe.encode_long's forward + backward on a synthetic one-hour recording (PASE+ in
eval mode, seeded weights, 57.6 M samples at 16 kHz) at two window sizes, for the full sweep
(parameter gradients and dx) and the frozen one (dx only), against the whole-recording encode +
backward at the longest length it runs here (tried from --encode-lengths down; a length that
runs out of memory is reported and skipped).  Host clock around work that ends in a device
synchronise, one warm-up call per mode first; peak allocated memory per mode (reset before each
call, so it counts the plans a call allocates and the tensors it returns).  The card's name and
power limit are read in the same run.  Prints a table, and writes the results as JSON to --out
when given.

    python tools/gpu/long_grad_time.py [--precision 3xf16] [--seconds 3600] [--out f.json]
"""
import argparse
import json
import os
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


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def set_frozen(model, frozen):
    for _, p in model.named_parameters():
        p.requires_grad_(not frozen)
        p.grad = None


def timed(fn, reps):
    """(median seconds, peak allocated bytes) over reps calls after one warm-up."""
    fn()
    times, peak = [], 0
    for _ in range(reps):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        peak = max(peak, torch.cuda.max_memory_allocated())
    times.sort()
    return times[len(times) // 2], peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="3xf16")
    ap.add_argument("--seconds", type=int, default=3600)
    ap.add_argument("--windows", type=int, nargs="+", default=[1 << 20, 1 << 19])
    ap.add_argument("--encode-lengths", type=int, nargs="+",
                    default=[16_000_000, 8_000_000, 4_000_000])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "long_grad_time.py needs a GPU"
    model = wf_builder(dict(PASE_PLUS))
    torch.manual_seed(0)
    model = model.cuda().eval()
    model.precision = args.precision
    g = torch.Generator().manual_seed(1)
    L = args.seconds * 16000
    wav = (0.5 * torch.randn(L, generator=g)).cuda()
    rows = []

    def long_call(win):
        def run():
            x = wav.clone().requires_grad_(True)
            y = model.encode_long(x, win)
            y.backward(cot[win])
            for _, p in model.named_parameters():
                p.grad = None
        return run

    cot = {}
    for win in args.windows:
        with torch.no_grad():
            shape = model.extract_long(wav, window=win).shape
        cot[win] = torch.randn(shape, generator=g).cuda()
        for frozen in (False, True):
            set_frozen(model, frozen)
            t, peak = timed(long_call(win), args.reps)
            rows.append(dict(call="encode_long", window=win, samples=L,
                             sweep="frozen" if frozen else "full", s=t, peak_gb=peak / 1e9,
                             audio_s_per_s=L / 16000 / t))
            print(rows[-1], flush=True)
    del cot
    for n in args.encode_lengths:
        x0 = wav[:n].view(1, 1, -1)
        ok = True
        for frozen in (False, True):
            set_frozen(model, frozen)

            def run():
                x = x0.clone().requires_grad_(True)
                y, _ = model.encode(x)
                y.backward(torch.ones_like(y))
                for _, p in model.named_parameters():
                    p.grad = None
            try:
                t, peak = timed(run, args.reps)
            except (torch.cuda.OutOfMemoryError, RuntimeError, ValueError) as e:
                print("encode at %d samples: %s" % (n, str(e).splitlines()[0][:200]), flush=True)
                ok = False
                break
            rows.append(dict(call="encode", window=None, samples=n,
                             sweep="frozen" if frozen else "full", s=t, peak_gb=peak / 1e9,
                             audio_s_per_s=n / 16000 / t))
            print(rows[-1], flush=True)
        model._plans.clear()
        torch.cuda.empty_cache()
        if ok:
            break
    info = gpu_info()
    print("card: %s, precision %s" % (info, args.precision))
    print("| call | window | samples | sweep | s | audio-s/s | peak GB |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %d | %s | %.3f | %.0f | %.2f |" % (
            r["call"], r["window"], r["samples"], r["sweep"], r["s"], r["audio_s_per_s"],
            r["peak_gb"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=info, precision=args.precision, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
