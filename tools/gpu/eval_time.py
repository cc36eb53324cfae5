"""Time per batch of the PASE+ validation pass from the resident corpus: the reference-style eager
loop (trainer.py:282-337: forward under no_grad, then ``.item()`` on every worker's loss and on the
total, every batch) against pase_b200.graph.GraphedEvalStep (one replay per batch, one
device-to-host copy per pass), in blocks that alternate between the two in one process.

Workload: PASE+.cfg + workers+.cfg (11 workers), B=32, T=32000, the model in eval mode; batches
assembled by DeviceBatcher from the valid split of the seeded synthetic corpus of
tools/gpu/batch_time.py (int16 utterances of 3 to 9 s, the seven cached workers+ features in HBM),
lps / lps_long computed on the device, the PASE+ distortions with codec2 and chop off.  Runs in
3xf16 and bf16, with ``fuse_regression_loss`` off and on (the fused heads run only in 3xf16; in
bf16 the flag changes nothing).

Per mode and block of --batches batches (one pass): device ms/batch (CUDA events around the block
on the pass stream), host ms/batch (the Python time to issue the block; for the eager loop this
includes its synchronising .item() calls, for GraphedEvalStep it excludes the final losses()),
and wall ms/batch (issue plus losses() / the final synchronise).

Run from the repository root after build():  python tools/gpu/eval_time.py [--batches 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

import torch  # noqa: E402
from batch_time import corpus  # noqa: E402
from distortion_banks import PASE_PLUS_P, base_cfg, build_banks  # noqa: E402
from pase_b200 import functional as Fn  # noqa: E402
from pase_b200.batch import DeviceBatcher, WavPool  # noqa: E402
from pase_b200.distortions import config_distortions  # noqa: E402
from pase_b200.graph import GraphedEvalStep  # noqa: E402
from pase_b200.pase import eval_losses, pase  # noqa: E402
from pase_b200.utils import parse_workers  # noqa: E402
from test_train_step import WORKERS_PLUS  # noqa: E402
from train_time import Batches  # noqa: E402
from helpers import resolve_cfg  # noqa: E402

HOP = 160


def valid_split(root, cfg, cache, n):
    """A 'valid' split of the first n utterances of the corpus, its features where
    DeviceBatcher.from_train_opts(split='valid') looks for them."""
    with open(cfg) as fh:
        data = json.load(fh)
    data["valid"] = {"data": data["train"]["data"][:n]}
    vcfg = os.path.join(root, "cfg_valid.json")
    with open(vcfg, "w") as fh:
        json.dump(data, fh)
    os.symlink(os.path.join(cache, "train"), os.path.join(cache, "valid"))
    return vcfg


def run(precision, fuse, wavs, cache, dist, B, T, nb, blocks):
    Fn.set_precision(precision)
    torch.manual_seed(0)
    model = pase(frontend_cfg=resolve_cfg("cfg/frontend/PASE+.cfg"),
                 minions_cfg=parse_workers(WORKERS_PLUS))
    model.frontend.precision = precision
    model.fuse_regression_loss = fuse
    model = model.cuda().eval()
    batcher = DeviceBatcher.from_train_opts(WORKERS_PLUS, T, HOP, wavs, random_scale=True,
                                            trans_cache=cache, split="valid", distortions=dist)
    feed = Batches(batcher, B)
    ev = GraphedEvalStep(model, batcher, B, max_batches=nb)
    s = ev.stream

    def eager_pass():
        running = {}
        for _ in range(nb):
            with torch.no_grad():
                _, _, preds, labels = model(batcher(feed.next()))
                tot, losses = eval_losses(model, preds, labels)
            for name, loss in losses.items():
                running.setdefault(name, []).append(loss.item())
            running.setdefault("total", []).append(tot.item())
        return running

    def graphed_pass():
        ev.reset()
        for _ in range(nb):
            ev(feed.next())

    def block(issue, finish):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            t0 = time.perf_counter()
            e0.record(s)
            issue()
            e1.record(s)
            t1 = time.perf_counter()
            out = finish()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        return (e0.elapsed_time(e1) / nb, (t1 - t0) * 1e3 / nb, (t2 - t0) * 1e3 / nb), out

    with torch.cuda.stream(s):
        graphed_pass()                          # 3 eager batches, capture, replays
        ev.losses()
        eager_pass()
    res = {"eager": [], "graphed": []}
    last = {}
    for _ in range(blocks):
        box = {}
        t, last["eager"] = block(lambda: box.update(r=eager_pass()), lambda: box["r"])
        res["eager"].append(t)
        t, last["graphed"] = block(graphed_pass, ev.losses)
        res["graphed"].append(t)
    out = {"precision": precision, "fuse_regression_loss": fuse, "B": B, "T": T,
           "batches_per_block": nb, "blocks": blocks,
           "last_pass_mean_total": {m: statistics.mean(v["total"]) for m, v in last.items()}}
    for mode, rows in res.items():
        dev, host, wall = zip(*rows)
        out[mode] = {"device_ms_per_batch": statistics.median(dev),
                     "host_ms_per_batch": statistics.median(host),
                     "wall_ms_per_batch": statistics.median(wall),
                     "device_ms_blocks": [round(v, 3) for v in dev],
                     "host_ms_blocks": [round(v, 3) for v in host],
                     "wall_ms_blocks": [round(v, 3) for v in wall]}
    out["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    del ev, model, batcher
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20, help="batches per timed block (a pass)")
    ap.add_argument("--blocks", type=int, default=3, help="blocks per mode, alternated")
    ap.add_argument("--utts", type=int, default=160)
    ap.add_argument("--valid-utts", type=int, default=96)
    ap.add_argument("--precisions", default="3xf16,bf16")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--chunk", type=int, default=32000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device:", q or torch.cuda.get_device_name(), flush=True)
    with tempfile.TemporaryDirectory() as root:
        data_root, cfg, cache = corpus(root, a.utts)
        vcfg = valid_split(root, cfg, cache, a.valid_utts)
        banks = build_banks(os.path.join(root, "banks"))
        dcfg = base_cfg(banks)
        dcfg.update(PASE_PLUS_P)
        dist = config_distortions(device="cuda", **dcfg)
        wavs = WavPool(data_root, vcfg, "valid", placement="cuda")
        for p in a.precisions.split(","):
            for fuse in (False, True):
                print(json.dumps(run(p, fuse, wavs, cache, dist, a.batch, a.chunk, a.batches,
                                     a.blocks)), flush=True)


if __name__ == "__main__":
    main()
