"""Cost of the waveform gradient of the PASE+ encoder (B=32, T=32000, seeded weights and input),
per precision (3xf16 and bf16 by default).  Backward passes timed with CUDA events, each after an
untimed forward, the modes alternated round-robin after a warm-up:

  full          the existing backward (parameters need gradients, the input does not);
  full+dx       the same backward returning dx as well;
  frozen_eval   the data-gradient-only backward of a frozen encoder in eval mode;
  frozen_train  the same in train mode (BatchNorm batch statistics).

Also each launch of the sinc layer's input gradient (encoder._sinc_input_grad), replayed with
its recorded arguments: the bank, the banded operand, the haloed dy copy, the polyphase GEMM
(with its operand conversion) and the fold-back.  The card's name and power limit are read in
the same run.  Prints a table, and writes the results as JSON to --out when given.

    python tools/gpu/input_grad_time.py [--precision 3xf16 bf16] [--reps 20]
                                        [--out results/input_grad.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from pase_b200 import encoder as enc, ops, wf_builder  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512,
             "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1}
B, T = 32, 32000
MODES = ["full", "full+dx", "frozen_eval", "frozen_train"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def time_backwards(prec, reps, warmup):
    torch.manual_seed(0)
    model = wf_builder(dict(PASE_PLUS)).cuda()
    model.precision = prec
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(1)).cuda()
    cot = torch.randn(B, 256, T // 160, generator=torch.Generator().manual_seed(2)).cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}

    def one(mode):
        model.load_state_dict(state)
        model.zero_grad(set_to_none=True)
        frozen = mode.startswith("frozen")
        for _, p in model.named_parameters():     # Model.parameters() skips frozen ones
            p.requires_grad_(not frozen)
        model.train(mode != "frozen_eval")
        xr = x.clone().requires_grad_(mode != "full")
        loss = (model(xr) * cot).sum()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss.backward()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b)

    times = {m: [] for m in MODES}
    for i in range(warmup + reps):
        for m in MODES:
            t = one(m)
            if i >= warmup:
                times[m].append(t)
    return model, x, {m: median(v) for m, v in times.items()}


def time_sinc_launches(model, x, reps):
    """Replay every launch of one _sinc_input_grad call with its arguments."""
    for _, p in model.named_parameters():
        p.requires_grad_(False)
    model.train(True)
    xr = x.clone().requires_grad_(True)
    (model(xr) ** 2).mean().backward()
    plan = model._plan(B, T, x.device)
    params = dict(model.named_parameters())
    calls, real = [], ops.call

    def spy(name, *a):
        calls.append((name, a))
        return real(name, *a)
    ops.call = spy
    try:
        dx = torch.empty(B, 1, T, device="cuda")
        enc._sinc_input_grad(plan, model, lambda k: params[k].detach().reshape(-1), plan.geoms[0],
                             dx)
    finally:
        ops.call = real
    out = []
    for name, a in calls:
        for _ in range(3):
            real(name, *a)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            real(name, *a)
        e.record()
        torch.cuda.synchronize()
        out.append((name, 1000.0 * s.elapsed_time(e) / reps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["3xf16", "bf16"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "input_grad_time.py needs a GPU"
    res = {"gpu": gpu_info(), "B": B, "T": T, "precisions": {}}
    print("card:", res["gpu"])
    for prec in args.precision:
        model, x, bwd = time_backwards(prec, args.reps, args.warmup)
        sinc = time_sinc_launches(model, x, args.reps)
        res["precisions"][prec] = {"backward_ms": bwd, "sinc_input_grad_us": sinc}
        print("%s: backward ms (median of %d)" % (prec, args.reps))
        for m in MODES:
            print("  %-13s %8.3f" % (m, bwd[m]))
        print("  sinc input gradient launches (us per call):")
        for name, us in sinc:
            print("    %-24s %8.1f" % (name, us))
        print("    %-24s %8.1f" % ("total", sum(us for _, us in sinc)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
