"""WaveFe.extract_long / FeatureStream timings on one GPU: audio-seconds per second for a
synthetic one-hour 16 kHz recording (CPU-resident, staged through pinned memory) at two window
sizes, peak allocated memory against the window size, and per-push latency of a stream for
10 ms and 100 ms pushes.  Prints one JSON line per measurement.

    python tools/gpu/extract_long_time.py [--precision 3xf16] [--minutes 60]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

from detweights import fill_state_dict  # noqa: E402
from pase_b200 import wf_builder  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512,
             "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1}
SR = 16000


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="3xf16")
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--pushes", type=int, default=300)
    a = ap.parse_args()
    torch.manual_seed(0)
    m = wf_builder(dict(PASE_PLUS))
    m.load_state_dict(fill_state_dict(m.state_dict(), 11))
    m.precision = a.precision
    m = m.cuda().eval()
    print(json.dumps({"gpu": gpu_info(), "precision": m.resolved_precision()}), flush=True)

    L = int(a.minutes * 60 * SR) // 160 * 160
    x = torch.randn(L) * 0.5
    for window in (1 << 20, 1 << 21):
        m.extract_long(x[:4 * window], window=window)           # warm-up: plan, pool, pinned slots
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        y = m.extract_long(x, window=window)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        print(json.dumps({"what": "extract_long", "audio_s": L / SR, "window": window,
                          "frames": y.shape[2], "wall_s": round(dt, 3),
                          "audio_s_per_s": round(L / SR / dt, 1)}), flush=True)
        del y
    m._packed_plans.clear()
    xs = x[:10 * 60 * SR]
    for window in (81920, 1 << 19, 1 << 20, 1 << 21):
        m._packed_plans.clear()                 # each row measures a call from a cold model
        m._long_pool = None
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        y = m.extract_long(xs, window=window)
        torch.cuda.synchronize()
        print(json.dumps({"what": "peak_memory", "audio_s": xs.numel() / SR, "window": window,
                          "peak_allocated_MB": round((torch.cuda.max_memory_allocated() - base)
                                                     / 2 ** 20, 1),
                          "output_MB": round(y.numel() * 4 / 2 ** 20, 1)}), flush=True)
        del y
    for push_ms in (10, 100):
        n = SR * push_ms // 1000
        st = m.stream()
        lat, a0 = [], 0
        for i in range(a.pushes + 200):
            t0 = time.perf_counter()
            f = st.push(x[a0:a0 + n])
            torch.cuda.synchronize()
            if i >= 200:                                          # past the first tail
                lat.append((time.perf_counter() - t0) * 1e3)
            a0 += n
        st.finish()
        lat.sort()
        print(json.dumps({"what": "stream_push", "push_ms": push_ms, "pushes": len(lat),
                          "median_ms": round(lat[len(lat) // 2], 3),
                          "p90_ms": round(lat[int(len(lat) * 0.9)], 3),
                          "max_ms": round(lat[-1], 3)}), flush=True)


if __name__ == "__main__":
    main()
