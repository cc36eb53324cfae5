"""StreamPool round times on one GPU: PASE+ eval, N live streams in {1, 16, 64, 256} fed 10 ms
(160-sample) or 100 ms (1600-sample) pushes.  Per case: the median and p90 of the synchronised
round time (one push() serving every stream) over --rounds rounds after warm-up, the same
rounds served by N independent FeatureStreams (each a one-stream pool whose plan holds one
window's longest segment) pushed one after another (the "seq" columns, over fewer rounds when N
is large: they are N times slower), whether the two gave equal frames, and, per push size, the
largest N whose median round stays below the push duration (real-time capacity).  The card's
name and power limit are read in the same run.  Prints one JSON line per measurement.

    python tools/gpu/stream_pool_time.py [--precisions 3xf16,bf16] [--rounds 300]
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
from pase_b200 import encoder as enc  # noqa: E402
from pase_b200 import ops  # noqa: E402

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


def pct(v, q):
    v = sorted(v)
    return round(v[min(len(v) - 1, int(len(v) * q))], 3)


def case(m, N, push, rounds, seq_rounds):
    warm = -(-(enc.tail_length(m.cfg) + enc.receptive_field(m.cfg)[1]) // push) + 5
    total = warm + rounds
    xs = torch.randn(N, push * total, generator=torch.Generator().manual_seed(N + push)) * 0.5
    pool = m.streams(N)
    ids = [pool.open() for _ in range(N)]
    sts = [m.stream() for _ in range(N)]
    blk = lambda k, r: xs[k, r * push:(r + 1) * push]            # noqa: E731
    for r in range(warm):                                          # past every stream's tail
        pool.push({i: blk(k, r) for k, i in enumerate(ids)})
        for k, st in enumerate(sts):
            st.push(blk(k, r))
    torch.cuda.synchronize()
    t_pool, t_seq, equal = [], [], True
    for r in range(warm, total):
        n0 = ops.launch_count
        t0 = time.perf_counter()
        res = pool.push({i: blk(k, r) for k, i in enumerate(ids)})
        torch.cuda.synchronize()
        t_pool.append((time.perf_counter() - t0) * 1e3)
        launches = ops.launch_count - n0
        if r < warm + seq_rounds:
            t0 = time.perf_counter()
            outs = [st.push(blk(k, r)) for k, st in enumerate(sts)]
            torch.cuda.synchronize()
            t_seq.append((time.perf_counter() - t0) * 1e3)
            equal &= all(torch.equal(res[i], o) for i, o in zip(ids, outs))
    return {"what": "round", "precision": m.resolved_precision(), "streams": N,
            "push_samples": push, "push_ms": push * 1000 / SR, "rounds": len(t_pool),
            "pool_median_ms": pct(t_pool, 0.5), "pool_p90_ms": pct(t_pool, 0.9),
            "seq_rounds": len(t_seq), "seq_median_ms": pct(t_seq, 0.5),
            "seq_p90_ms": pct(t_seq, 0.9), "equal": bool(equal),
            "launches_per_round": launches,
            "plan_MB": round(pool.plan.nbytes() / 2 ** 20, 1),
            "arena_MB": round(pool.ring.numel() * 4 / 2 ** 20, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="3xf16,bf16")
    ap.add_argument("--streams", default="1,16,64,256")
    ap.add_argument("--pushes", default="160,1600")
    ap.add_argument("--rounds", type=int, default=300)
    ap.add_argument("--seq-budget", type=int, default=3000,
                    help="FeatureStream pushes timed per case (rounds = budget / N, >= 10)")
    a = ap.parse_args()
    torch.manual_seed(0)
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for prec in a.precisions.split(","):
        m = wf_builder(dict(PASE_PLUS))
        m.load_state_dict(fill_state_dict(m.state_dict(), 11))
        m.precision = prec
        m = m.cuda().eval()
        for push in [int(p) for p in a.pushes.split(",")]:
            cap = None
            for N in [int(n) for n in a.streams.split(",")]:
                r = case(m, N, push, a.rounds, min(a.rounds, max(10, a.seq_budget // N)))
                print(json.dumps(r), flush=True)
                if r["pool_median_ms"] < r["push_ms"]:
                    cap = N
                m._packed_plans.clear()
                torch.cuda.empty_cache()
            print(json.dumps({"what": "real_time_capacity", "precision": prec,
                              "push_samples": push, "largest_N_measured": cap,
                              "of": a.streams}), flush=True)
    print(json.dumps({"gpu_end": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
