"""Cost of the BatchNorm column statistics in the wgmma NT GEMM epilogue, per launch of the PASE+
training step (B=32, T=32000, seeded weights and input).  One eager forward + backward records
the arguments of every `pase_tc_gemm_nt` call; each forward call is then replayed with its
statistics (`colsum` / `colsumsq`, into separate zeroed sums) and without them (NULL), the two
alternated in blocks of launches timed with CUDA events after a warm-up, and each backward
(data-gradient) call as it ran, so a forward conv GEMM can be set against its dgrad partner of
nearly the same shape.  Every call covers bulk + tail launches (nt_plan).  The card's name and
power limit are read in the same run.  Prints a table, and writes the results as JSON to --out
when given.

    python tools/gpu/nt_stats_time.py [--precision 3xf16] [--blocks 10] [--per-block 10]
                                      [--out results/nt_stats.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from pase_b200 import ops, wf_builder  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512,
             "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1}
B, T = 32, 32000
FWD = ["sinc", "block1", "block2", "block3", "block4", "block5", "block6", "block7", "qrnn",
       "W+skips"]
BWD = ["W+skips", "qrnn", "block7", "block6", "block5", "block4", "block3", "block2", "block1"]
# pase_tc_gemm_nt argument positions (include/pase_b200.h, stream excluded)
I_M, I_N, I_K, I_CS, I_CQ = 9, 10, 11, 19, 20


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def record_step(prec):
    """(forward calls, backward calls): argument tuples of every pase_tc_gemm_nt call of one
    eager training step, the tensors kept alive by the tuples."""
    torch.manual_seed(0)
    model = wf_builder(dict(PASE_PLUS)).cuda().train()
    model.precision = prec
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(1)).cuda()
    calls, real = [], ops.call

    def spy(name, *a):
        if name == "pase_tc_gemm_nt":
            calls.append(a)
        return real(name, *a)
    ops.call = spy
    try:
        y = model(x)
        n_fwd = len(calls)
        y.square().mean().backward()
        torch.cuda.synchronize()
    finally:
        ops.call = real
    return calls[:n_fwd], calls[n_fwd:]


def time_calls(variants, blocks, per_block, warmup=5):
    """variants: list of argument tuples.  -> per variant, the median over `blocks` blocks of the
    mean launch time (us) of `per_block` back-to-back calls; the variants alternate block by
    block."""
    for a in variants:
        for _ in range(warmup):
            ops.call("pase_tc_gemm_nt", *a)
    torch.cuda.synchronize()
    times = [[] for _ in variants]
    for _ in range(blocks):
        for i, a in enumerate(variants):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(per_block):
                ops.call("pase_tc_gemm_nt", *a)
            e.record()
            e.synchronize()
            times[i].append(s.elapsed_time(e) * 1e3 / per_block)
    return [sorted(t)[len(t) // 2] for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="3xf16")
    ap.add_argument("--blocks", type=int, default=10)
    ap.add_argument("--per-block", type=int, default=10)
    ap.add_argument("--out", default=None, help="JSON file for the results")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "nt_stats_time.py needs a GPU"
    torch.cuda.set_device(0)
    info = gpu_info()
    fwd, bwd = record_step(args.precision)
    fnames = FWD if len(fwd) == len(FWD) else ["fwd%d" % i for i in range(len(fwd))]
    bnames = BWD if len(bwd) == len(BWD) else ["bwd%d" % i for i in range(len(bwd))]
    rows = []
    for name, a in zip(fnames, fwd):
        M, N, K = a[I_M], a[I_N], a[I_K]
        flop = 2.0 * M * N * K
        row = {"launch": name + " fwd", "M": M, "N": N, "K": K}
        if a[I_CS] is not None:
            off = list(a)
            off[I_CS] = off[I_CQ] = None
            on = list(a)
            on[I_CS] = torch.zeros_like(a[I_CS])
            on[I_CQ] = torch.zeros_like(a[I_CQ])
            t_on, t_off = time_calls([tuple(on), tuple(off)], args.blocks, args.per_block)
            row.update(us_stats=t_on, us_no_stats=t_off, tflops_stats=flop / t_on * 1e-6,
                       tflops_no_stats=flop / t_off * 1e-6)
        else:
            (t,) = time_calls([a], args.blocks, args.per_block)
            row.update(us=t, tflops=flop / t * 1e-6)
        rows.append(row)
    for name, a in zip(bnames, bwd):
        M, N, K = a[I_M], a[I_N], a[I_K]
        (t,) = time_calls([a], args.blocks, args.per_block)
        rows.append({"launch": name + " dgrad", "M": M, "N": N, "K": K, "us": t,
                     "tflops": 2.0 * M * N * K / t * 1e-6})
    res = {"gpu": info, "device": torch.cuda.get_device_name(0), "precision": args.precision,
           "B": B, "T": T, "blocks": args.blocks, "per_block": args.per_block, "launches": rows}
    print("# %s | %s | %s, %d x %d launches per variant" % (res["device"], info, args.precision,
                                                           args.blocks, args.per_block))
    print("| launch | M x N x K | us stats | TFLOP/s | us no stats | TFLOP/s |")
    print("|---|---|---:|---:|---:|---:|")
    for r in rows:
        shape = "%d x %d x %d" % (r["M"], r["N"], r["K"])
        if "us_stats" in r:
            print("| %s | %s | %.1f | %.0f | %.1f | %.0f |" % (
                r["launch"], shape, r["us_stats"], r["tflops_stats"], r["us_no_stats"],
                r["tflops_no_stats"]))
        else:
            print("| %s | %s | %.1f | %.0f | | |" % (r["launch"], shape, r["us"], r["tflops"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
