"""ms per B=64, T=48000 batch of the on-device distortions (pase_b200/distortions.py), with CUDA
events, at the PASE+ probabilities (cfg/distortions/pase+.cfg, codec2 and chop off) and with
every stage at p = 1.  Banks: the seeded synthetic ones of tests/golden/distortion_banks.py
(three IRs up to 24000 taps, 100-103-tap FIRs).  Run from the repository root after build():
    python tools/gpu/distortions_time.py [--iters 50]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import torch  # noqa: E402
from distortion_banks import PASE_PLUS_P, base_cfg, build_banks, make_chunk  # noqa: E402
from pase_b200.distortions import config_distortions  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=48000)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        q = torch.cuda.get_device_name()
    print("device:", q)
    all_p = dict(reverb_p=1.0, overlap_p=1.0, overlap_reverb=True, noises_p=1.0, clip_p=1.0,
                 bandrop_p=1.0, downsample_p=1.0)
    with tempfile.TemporaryDirectory() as root:
        paths = build_banks(root)
        x = torch.from_numpy(make_chunk(a.B, a.T, 0)).view(a.B, 1, a.T).cuda()
        for label, over in (("pase+ probabilities", PASE_PLUS_P), ("every stage p=1", all_p)):
            cfg = base_cfg(paths)
            cfg.update(over)
            dist = config_distortions(device="cuda", **cfg)
            plans = [dist.plan(a.B, a.T) for _ in range(a.iters)]
            t0 = time.perf_counter()
            for _ in range(20):
                dist.plan(a.B, a.T)
            plan_ms = (time.perf_counter() - t0) / 20 * 1e3
            for p in plans[:5]:
                dist.apply(x, p)
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for p in plans:
                dist.apply(x, p)
            ev1.record()
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1) / a.iters
            print("%-20s B=%d T=%d: %.3f ms/batch on the device (upload + kernels), host planner "
                  "%.3f ms/batch" % (label, a.B, a.T, ms, plan_ms))


if __name__ == "__main__":
    main()
