#!/usr/bin/env python
"""Per-launch table of the tensor-core GEMMs of one PASE+ encoder step (B=32, T=32000):
shape, time (CUDA events around each launch, eager), fp32-equivalent TFLOP/s.  Meant for
A/B runs of kernel variants selected by PASE_B200_* environment switches (read once per
process by the library).  Needs a GPU; `--precision`
as in bench.py.  Not part of the library; measurement helper only.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench import PASE_PLUS, B_PER_GPU, T_CHUNK          # noqa: E402  (workload definition)
from pase_b200 import ops, wf_builder                    # noqa: E402


def shape_of(name, a):
    """(kind, M/I, N/J, K/rows, flop) from the C-ABI argument list (include/pase_b200.h)."""
    if name == "pase_tc_gemm_nt":
        M, N, K = a[9], a[10], a[11]
        return "NT", M, N, K, 2.0 * M * N * K
    if name == "pase_tc_gemm_tn":
        I, J, groups, rpg = a[12], a[13], a[14], a[15]
        return "TN", I, J, groups * rpg, 2.0 * I * J * groups * rpg
    if name == "pase_gemm_nt":
        M, N, K = a[6], a[7], a[8]
        return "nt(ffma)", M, N, K, 2.0 * M * N * K
    I, J, groups, rpg = a[10], a[11], a[12], a[13]
    return "tn(ffma)", I, J, groups * rpg, 2.0 * I * J * groups * rpg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="3xtf32", choices=["fp32", "3xtf32", "tf32"])
    ap.add_argument("--batch", type=int, default=B_PER_GPU)
    ap.add_argument("--repeats", type=int, default=3, help="instrumented steps (min is kept)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = wf_builder(dict(PASE_PLUS)).to(dev).train()
    model.precision = args.precision
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, fused=True)
    x = torch.randn(args.batch, 1, T_CHUNK, device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        model(x).square().mean().backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    names = ("pase_gemm_nt", "pase_gemm_tn", "pase_tc_gemm_nt", "pase_tc_gemm_tn")
    real_call = ops.call
    best = None
    for _ in range(args.repeats):
        recs = []

        def spy(name, *a):
            if name not in names:
                return real_call(name, *a)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = real_call(name, *a)
            e.record()
            recs.append((name, a, s, e))
            return r
        ops.call = spy
        try:
            step()
            torch.cuda.synchronize()
        finally:
            ops.call = real_call
        rows = [shape_of(n, a) + (s.elapsed_time(e),) for n, a, s, e in recs]
        if best is None:
            best = rows
        else:
            best = [b if b[5] <= r[5] else r for b, r in zip(best, rows)]
    env = {k: v for k, v in os.environ.items() if k.startswith("PASE_B200_")}
    print("# GEMM launches of one PASE+ step (B=%d, T=%d, %s), switches %s" %
          (args.batch, T_CHUNK, args.precision, env or "{}"))
    print()
    print("| # | kind | M / I | N / J | K / rows | ms | TFLOP/s |")
    print("|---|---|---:|---:|---:|---:|---:|")
    tot_ms = tot_fl = 0.0
    for i, (kind, m, n, k, fl, ms) in enumerate(best):
        print("| %d | %s | %d | %d | %d | %.4f | %.1f |" % (i, kind, m, n, k, ms, fl / ms / 1e9))
        tot_ms += ms
        tot_fl += fl
    print()
    print("total: %.3f ms, %.1f TFLOP/s" % (tot_ms, tot_fl / tot_ms / 1e9))


if __name__ == "__main__":
    main()
