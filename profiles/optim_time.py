"""Time pase_adam_flat at the workers+ layout (13 segments, 29.7 M parameters, each segment
padded to a multiple of 4 as FlatAdam lays it out) with CUDA events, for an all-Adam and an
all-RAdam table; with --baseline, also a second build of the library (e.g. the previous
commit's) on the all-Adam table, alternating with this one, and its all-Adam outputs compared
bit for bit with this build's.

    python profiles/optim_time.py [--baseline path/to/libpase_b200.so] [--out result.json]

The update reads p, g, m, v and writes p, m, v: 7 x 4 bytes per element.
"""
import argparse
import ctypes
import json
import os
import struct
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pase_b200 import _lib  # noqa: E402

WORKERS_PLUS = [7832896, 131841, 131841, 8857537, 5597973, 5597973, 281928, 281928, 281928,
                281928, 136209, 173988, 87636]


def seg_table(algo):
    raw, off = b"", 0
    for k, size in enumerate(WORKERS_PLUS):
        end = off + (size + 3) // 4 * 4
        raw += struct.pack("<qqffffffq", off, end, 5e-4, 0.9, 0.999, 1e-8, 0.0, float(algo), k)
        off = end
    return torch.frombuffer(bytearray(raw), dtype=torch.int64).cuda(), off


def launcher(L, bufs, table, steps, n):
    fn = L.pase_adam_flat
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_long, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p]
    args = [b.data_ptr() for b in bufs] + [n, table.data_ptr(), len(WORKERS_PLUS),
                                           steps.data_ptr(), 1.0]

    def run():
        rc = fn(*args, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc
    run.keep = (bufs, table, steps)            # the pointers above stay valid
    return run


def fresh(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(n, device="cuda", generator=g),
            torch.randn(n, device="cuda", generator=g) * 1e-2,
            torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", default=None)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    cur = _lib.lib()
    libs = {"this": cur}
    if a.baseline:
        libs["baseline"] = ctypes.CDLL(os.path.abspath(a.baseline))
    t_adam, n = seg_table(0)
    t_radam, _ = seg_table(1)
    steps = torch.full((len(WORKERS_PLUS),), 10.0, device="cuda")
    cases = {"adam_this": ("this", t_adam), "radam_this": ("this", t_radam)}
    if a.baseline:
        cases["adam_baseline"] = ("baseline", t_adam)
    runs = {}
    for name, (lib, tab) in cases.items():
        bufs = fresh(n, 1)
        runs[name] = launcher(libs[lib], bufs, tab, steps, n)
    # outputs: identical inputs, 12 updates with growing step counts
    outs = {}
    for name in ("adam_this", "adam_baseline", "radam_this"):
        if name not in cases:
            continue
        lib, tab = cases[name]
        bufs, st = fresh(n, 2), torch.zeros_like(steps)
        run = launcher(libs[lib], bufs, tab, st, n)
        for _ in range(12):
            st += 1.0
            run()
        outs[name] = bufs
    torch.cuda.synchronize()
    res = {"elements": n, "bytes_per_launch": 7 * 4 * n, "launches_per_window": a.launches}
    if "adam_baseline" in outs:
        res["adam_bit_equal_to_baseline"] = all(
            torch.equal(x, y) for x, y in zip(outs["adam_this"], outs["adam_baseline"]))
    res["radam_finite"] = bool(torch.isfinite(outs["radam_this"][0]).all())
    for run in runs.values():                 # warm-up
        for _ in range(20):
            run()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for name, run in runs.items():        # alternate the builds and tables
            ev0.record()
            for _ in range(a.launches):
                run()
            ev1.record()
            ev1.synchronize()
            times[name].append(ev0.elapsed_time(ev1) * 1e3 / a.launches)
    for name, ts in times.items():
        ts = sorted(ts)
        res[name + "_us"] = {"median": ts[len(ts) // 2], "min": ts[0], "max": ts[-1]}
        res[name + "_GBps"] = res["bytes_per_launch"] / (ts[len(ts) // 2] * 1e-6) / 1e9
    res["device"] = torch.cuda.get_device_name(0)
    try:
        import subprocess
        res["power_limit"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit"] = "unknown"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
