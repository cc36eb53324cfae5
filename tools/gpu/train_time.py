"""Time per step of a PASE+ training step from the resident corpus, eager loop against
pase_b200.graph.GraphedTrainStep, in blocks that alternate between the two in one process.

Workload: PASE+.cfg + workers+.cfg (12 workers), B=32, T=32000; batches assembled by
DeviceBatcher on the seeded synthetic corpus tools/gpu/batch_time.py builds (int16 utterances of
3 to 9 s, the seven cached workers+ features in HBM), lps / lps_long computed on the device, the
PASE+ distortions with codec2 and chop off; FlatAdam with one group per module, the encoder
bound; an lr change for every group before every step (a poly schedule).

Per mode and block: device ms/step (CUDA events around the block on the step stream), host
ms/step (the Python time to issue the block, no synchronise inside it; for GraphedTrainStep this
includes its waits for a free staging table, i.e. the device's back-pressure once the host is two
steps ahead), wall ms/step (issue plus the final synchronise), and the issue cost: the host time
of one call made with the device idle (synchronised before each call), which is what the host
spends per step.  Both modes run on the same model, engine and batcher, one after the other on
one stream.

Run from the repository root after build():  python tools/gpu/train_time.py [--steps 20]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402
from batch_time import corpus  # noqa: E402
from distortion_banks import PASE_PLUS_P, base_cfg, build_banks  # noqa: E402
from pase_b200 import functional as Fn  # noqa: E402
from pase_b200.batch import DeviceBatcher, WavPool  # noqa: E402
from pase_b200.distortions import config_distortions  # noqa: E402
from pase_b200.graph import GraphedTrainStep  # noqa: E402
from pase_b200.optim import FlatAdam  # noqa: E402
from pase_b200.pase import pase, total_loss  # noqa: E402
from pase_b200.utils import parse_workers  # noqa: E402
from test_train_step import WORKERS_PLUS  # noqa: E402
from helpers import resolve_cfg  # noqa: E402

HOP = 160


class Batches:
    """Shuffled index lists, epoch after epoch, with the batcher reset at each epoch."""

    def __init__(self, batcher, B, seed=0):
        self.batcher, self.B, self.rng, self.queue = batcher, B, np.random.RandomState(seed), []

    def next(self):
        if not self.queue:
            self.batcher.reset()
            n = len(self.batcher.wavs)
            perm = self.rng.permutation(n).tolist()
            self.queue = [perm[j:j + self.B] for j in range(0, n - self.B + 1, self.B)]
        return self.queue.pop(0)


def run(precision, wavs, cache, dist, B, T, steps, blocks):
    Fn.set_precision(precision)
    torch.manual_seed(0)
    model = pase(frontend_cfg=resolve_cfg("cfg/frontend/PASE+.cfg"),
                 minions_cfg=parse_workers(WORKERS_PLUS))
    model.frontend.precision = precision
    model = model.cuda().train()
    groups = [{"params": list(model.frontend.parameters())}]
    groups += [{"params": list(w.parameters())} for w in
               list(model.classification_workers) + list(model.regression_workers)]
    engine = FlatAdam(groups, lr=1e-4).bind_encoder(model.frontend)
    batcher = DeviceBatcher.from_train_opts(WORKERS_PLUS, T, HOP, wavs, random_scale=True,
                                            trans_cache=cache, distortions=dist)
    feed = Batches(batcher, B)
    step = GraphedTrainStep(model, engine, batcher, B)
    k = [0]

    def poly():
        for gi, g in enumerate(engine.param_groups):
            g["lr"] = 1e-4 * (1.0 - (k[0] % 1000) / 1000.0) ** 0.9
        k[0] += 1

    def eager():
        poly()
        engine.zero_grad(set_to_none=True)
        batch = batcher(feed.next())
        _, _, preds, labels = model(batch)
        tot, _ = total_loss(model, preds, labels)
        tot.backward()
        engine.step()

    def graphed():
        poly()
        step(feed.next())

    def block(fn):
        s = step.stream
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            t0 = time.perf_counter()
            e0.record(s)
            for _ in range(steps):
                fn()
            e1.record(s)
            t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        return e0.elapsed_time(e1) / steps, (t1 - t0) * 1e3 / steps, (t2 - t0) * 1e3 / steps

    def issue(fn):
        ms = []
        with torch.cuda.stream(step.stream):
            for _ in range(steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                ms.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        return statistics.median(ms)

    with torch.cuda.stream(step.stream):
        for _ in range(5):                      # GraphedTrainStep: 3 eager, capture, replay
            graphed()
        for _ in range(3):
            eager()
    res = {"eager": [], "graphed": []}
    for _ in range(blocks):
        res["eager"].append(block(eager) + (issue(eager),))
        res["graphed"].append(block(graphed) + (issue(graphed),))
    out = {"precision": precision, "B": B, "T": T, "steps_per_block": steps, "blocks": blocks,
           "last_losses": step.losses()}
    for mode, rows in res.items():
        dev, host, wall, cost = zip(*rows)
        out[mode] = {"device_ms_per_step": statistics.median(dev),
                     "host_ms_per_step": statistics.median(host),
                     "wall_ms_per_step": statistics.median(wall),
                     "host_issue_ms_per_step": statistics.median(cost),
                     "device_ms_blocks": [round(v, 3) for v in dev],
                     "host_ms_blocks": [round(v, 3) for v in host]}
    out["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    del step, model, engine, batcher
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="steps per timed block")
    ap.add_argument("--blocks", type=int, default=3, help="blocks per mode, alternated")
    ap.add_argument("--utts", type=int, default=160)
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
        banks = build_banks(os.path.join(root, "banks"))
        dcfg = base_cfg(banks)
        dcfg.update(PASE_PLUS_P)
        dist = config_distortions(device="cuda", **dcfg)
        wavs = WavPool(data_root, cfg, "train", placement="cuda")
        for p in a.precisions.split(","):
            print(json.dumps(run(p, wavs, cache, dist, a.batch, a.chunk, a.steps, a.blocks)),
                  flush=True)


if __name__ == "__main__":
    main()
