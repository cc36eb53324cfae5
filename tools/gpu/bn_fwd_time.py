"""Time every forward BatchNorm/PReLU launch (`pase_bn_prelu_pad_fwd`) of the PASE+ training
step (B=32, T=32000, seeded weights and input), blocks 0-7, in each precision asked for.

One eager forward records the arguments of every call; each call is then replayed with CUDA
events, in blocks of back-to-back launches after a warm-up, and the median block gives the time
per launch.  Bytes moved per launch: y read, the operand written (fp32 4 B, + 4 B with the
3xTF32 residual twin; bf16 2 B; fp16 pair 4 B per element, halo rows included) and the pooled
dense-skip values written (4 B each); the rate is set against the H100 SXM's 3.35 TB/s.  The
card's name and power limit are read in the same run.

With --baseline (a second build of the library, e.g. the previous commit's), the two builds
alternate block by block, and each call's outputs (operand and pool) from both builds are
compared bit for bit on the same inputs.

    python tools/gpu/bn_fwd_time.py [--precision 3xf16 bf16] [--baseline path/to/libpase_b200.so]
                                    [--blocks 10] [--per-block 10] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from pase_b200 import _lib, ops, wf_builder  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512,
             "denseskips": True, "norm_out": True, "rnn_pool": True, "rnn_layers": 1}
B, T = 32, 32000
NAME = "pase_bn_prelu_pad_fwd"
HBM_TBS = 3.35
# argument positions (include/pase_b200.h, stream excluded)
I_Y, I_YBF, I_N, I_T, I_C, I_DST, I_LO, I_FMT, I_PADL, I_PADR = 0, 1, 3, 4, 5, 9, 10, 11, 14, 15
I_POOL, I_PD, I_PT = 16, 19, 20


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the query is informational only
        out = "unavailable: %s" % e
    return out.splitlines()[0] if out else out


def record_forward(prec):
    """Argument tuples of every pase_bn_prelu_pad_fwd call of one eager training forward, the
    tensors kept alive by the tuples."""
    torch.manual_seed(0)
    model = wf_builder(dict(PASE_PLUS)).cuda().train()
    model.precision = prec
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(1)).cuda()
    calls, real = [], ops.call

    def spy(name, *a):
        if name == NAME:
            calls.append(a)
        return real(name, *a)
    ops.call = spy
    try:
        model(x)
        torch.cuda.synchronize()
    finally:
        ops.call = real
    return calls, model


def bytes_moved(a):
    N, Tn, C = a[I_N], a[I_T], a[I_C]
    Tp = Tn + a[I_PADL] + a[I_PADR]
    y = N * Tn * C * (2 if a[I_YBF] else 4)
    fmt = a[I_FMT]
    per = {0: 8 if a[I_LO] is not None else 4, 1: 2, 2: 4}[fmt]
    dst = N * Tp * C * per
    pool = N * a[I_PT] * C * 4 if (a[I_POOL] is not None and a[I_PD] > 0) else 0
    return y, dst, pool


def launcher(L, a):
    """A no-argument function launching `a` through library handle L."""
    ret, params = _lib.PROTOS[NAME]
    cargs = [_lib._ptr(v, t, NAME, pn) if p else v for (t, p, pn), v in zip(params, a)]
    fn = getattr(L, NAME)
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p if p else _lib._CTYPES[t] for (t, p, _) in params]

    def run():
        rc = fn(*cargs, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, (rc, _lib.last_error())
    return run


def time_runs(runs, blocks, per_block, warmup=5):
    """-> per run, the median over `blocks` blocks of the mean launch time (us) of `per_block`
    back-to-back launches; the runs alternate block by block."""
    for r in runs:
        for _ in range(warmup):
            r()
    torch.cuda.synchronize()
    times = [[] for _ in runs]
    for _ in range(blocks):
        for i, r in enumerate(runs):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(per_block):
                r()
            e.record()
            e.synchronize()
            times[i].append(s.elapsed_time(e) * 1e3 / per_block)
    return [sorted(t)[len(t) // 2] for t in times]


def outputs(run, a):
    """Run once on zeroed outputs; -> clones of the operand (+ lo) and pool."""
    outs = [a[i] for i in (I_DST, I_LO, I_POOL) if a[i] is not None]
    for o in outs:
        o.zero_()
    run()
    torch.cuda.synchronize()
    return [o.clone() for o in outs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["3xf16", "bf16"])
    ap.add_argument("--baseline", default=None)
    ap.add_argument("--blocks", type=int, default=10)
    ap.add_argument("--per-block", type=int, default=10)
    ap.add_argument("--out", default=None, help="JSON file for the results")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bn_fwd_time.py needs a GPU"
    torch.cuda.set_device(0)
    info = gpu_info()
    libs = {"this": _lib.lib()}
    if args.baseline:
        libs["baseline"] = ctypes.CDLL(os.path.abspath(args.baseline))
    res = {"gpu": info, "device": torch.cuda.get_device_name(0), "B": B, "T": T,
           "blocks": args.blocks, "per_block": args.per_block, "launches": []}
    print("# %s | %s | %d x %d launches per build and call" % (res["device"], info,
                                                                args.blocks, args.per_block))
    for prec in args.precision:
        calls, model = record_forward(prec)
        print("\n## %s\n" % prec)
        print("| block | T x C | pool_d | MB moved | " + " | ".join(
            "us %s | TB/s %s" % (k, k) for k in libs) + " | bit-equal |")
        print("|---|---|---:|---:|" + "---:|---:|" * len(libs) + "---|")
        for l, a in enumerate(calls):
            runs = [launcher(L, a) for L in libs.values()]
            same = None
            if len(runs) > 1:
                ref = outputs(runs[0], a)
                same = all(torch.equal(x.view(torch.uint8), y.view(torch.uint8))
                           for x, y in zip(ref, outputs(runs[1], a)))
            us = time_runs(runs, args.blocks, args.per_block)
            yb, db, pb = bytes_moved(a)
            tot = yb + db + pb
            row = {"precision": prec, "block": l, "N": a[I_N], "T": a[I_T], "C": a[I_C],
                   "pool_d": a[I_PD], "pool_T": a[I_PT], "bytes_y": yb, "bytes_dst": db,
                   "bytes_pool": pb, "bit_equal": same}
            for k, t in zip(libs, us):
                row["us_" + k] = t
                row["tbs_" + k] = tot / t * 1e-6
            res["launches"].append(row)
            print("| %d | %d x %d | %d | %.1f | %s | %s |" % (
                l, a[I_T], a[I_C], a[I_PD], tot / 1e6,
                " | ".join("%.1f | %.2f (%.0f%%)" % (t, tot / t * 1e-6,
                                                     100 * tot / t * 1e-6 / HBM_TBS) for t in us),
                "-" if same is None else ("yes" if same else "NO")))
        del calls, model
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
