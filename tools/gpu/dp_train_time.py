"""Weak scaling of the data-parallel captured PASE+ training step (GraphedTrainStep(group=...))
over the GPUs of one node: the peer-memory update (FlatAdam(peer_dp=True), one replay per step)
against the NCCL fallback (plain FlatAdam, two replays with the all-reduce between them),
alternated in one session.

Workloads (PASE+.cfg + workers+.cfg, every head; the seeded synthetic corpus of
tools/gpu/batch_time.py; the banks of tests/golden/distortion_banks.py, PASE+ distortions with
codec2 and chop off; FlatAdam with one group per module):
    c3  B=32 per GPU, T=32000, 3xf16 and bf16
    c4  B=64 per GPU, T=48000, bf16
Each rank draws its batches from its DistributedSampler shard (shuffle, drop_last, shared seed
and epoch) and its own generator triple.

Per run: device ms/step (CUDA events around a block of steps on the step stream, the slowest
rank), global samples/s, host issue ms/step (one call with the device idle, median), peak
memory (torch's allocator, the largest rank, plus the peer-mapped buffers), and the weak-scaling
efficiency against N=1 (device ms at N=1 over device ms at N).  Before the data-parallel runs
every rank builds and replays the step alone; an out-of-memory there is reported as the result
of the workload on every rank, and the data-parallel runs of that workload are skipped.

Run from the repository root after build():
    python tools/gpu/dp_train_time.py [--gpus 1,2,4,8] [--steps 20] [--reps 2]
It builds the corpus once, launches ``torchrun --standalone --nproc_per_node=N`` for each N the
machine has, waits for it, and prints one JSON line per run.
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

import random  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

HOP = 160
WORKLOADS = {"c3": (32, 32000, ("3xf16", "bf16")), "c4": (64, 48000, ("bf16",))}


def _triple(s):
    return (random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


class Shard:
    """Rank `rank`'s index lists, epoch after epoch (DistributedSampler, then BatchSampler),
    with the batcher reset at each epoch."""

    def __init__(self, batcher, B, world, rank, seed=0):
        from torch.utils.data import DistributedSampler
        self.batcher, self.queue, self.epoch = batcher, [], 0
        self.sampler = DistributedSampler(range(len(batcher.wavs)), num_replicas=world, rank=rank,
                                          shuffle=True, seed=seed, drop_last=True)
        self.B = B

    def next(self):
        from torch.utils.data import BatchSampler
        if not self.queue:
            self.sampler.set_epoch(self.epoch)
            self.epoch += 1
            self.batcher.reset()
            self.queue = [list(b) for b in BatchSampler(self.sampler, self.B, drop_last=True)]
        return self.queue.pop(0)


def build(args, precision, B, T, engine_kw, group):
    from distortion_banks import PASE_PLUS_P, base_cfg
    from pase_b200 import functional as Fn
    from pase_b200.batch import DeviceBatcher, WavPool
    from pase_b200.distortions import config_distortions
    from pase_b200.dp import broadcast_parameters_and_buffers
    from pase_b200.graph import GraphedTrainStep
    from pase_b200.optim import FlatAdam
    from pase_b200.pase import pase
    from pase_b200.utils import parse_workers
    from helpers import resolve_cfg
    from test_train_step import WORKERS_PLUS
    Fn.set_precision(precision)
    torch.manual_seed(0)
    model = pase(frontend_cfg=resolve_cfg("cfg/frontend/PASE+.cfg"),
                 minions_cfg=parse_workers(WORKERS_PLUS))
    model.frontend.precision = precision
    model = model.cuda().train()
    if group is not None:
        broadcast_parameters_and_buffers(model, group=group)
    groups = [{"params": list(model.frontend.parameters())}]
    groups += [{"params": list(w.parameters())} for w in
               list(model.classification_workers) + list(model.regression_workers)]
    engine = FlatAdam(groups, lr=1e-4, **engine_kw).bind_encoder(model.frontend)
    dcfg = base_cfg(json.load(open(os.path.join(args.root, "banks.json"))))
    dcfg.update(PASE_PLUS_P)
    wavs = WavPool(args.data_root, args.cfg, "train", placement="cuda")
    batcher = DeviceBatcher.from_train_opts(WORKERS_PLUS, T, HOP, wavs, random_scale=True,
                                            trans_cache=args.cache,
                                            distortions=config_distortions(device="cuda", **dcfg))
    step = GraphedTrainStep(model, engine, batcher, B, group=group)
    return model, engine, step


def release(engine):
    """Unmap the peers' buffers and free this rank's (every rank has finished with them)."""
    import torch.distributed as dist
    if engine._peer is None:
        return
    torch.cuda.synchronize()
    dist.barrier()
    engine._peer.close()
    for a in engine._peer.allocs.values():
        a.free()


def timed(step, feed, rng, steps, group):
    """-> (device ms/step of the slowest rank, host issue ms/step)."""
    import torch.distributed as dist
    for _ in range(5):                      # 3 eager, capture, replay
        step(feed.next(), rng)
    torch.cuda.synchronize()
    if group is not None:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(step.stream)
    for _ in range(steps):
        step(feed.next(), rng)
    e1.record(step.stream)
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / steps], device="cuda")
    issue = []
    for _ in range(min(steps, 10)):
        torch.cuda.synchronize()
        if group is not None:
            dist.barrier()
        t0 = time.perf_counter()
        step(feed.next(), rng)
        issue.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    if group is not None:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX, group=group)
    return float(ms), statistics.median(issue)


def peak_gb(extra_bytes, group):
    import torch.distributed as dist
    t = torch.tensor([torch.cuda.max_memory_allocated() + extra_bytes], dtype=torch.float64,
                     device="cuda")
    if group is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t) / 2 ** 30


def run_one(args, precision, B, T, mode, world, rank, group):
    kw = {"peer_dp": True} if mode == "peer" else {}
    torch.cuda.reset_peak_memory_stats()
    model, engine, step = build(args, precision, B, T, kw, group)
    feed = Shard(step.batcher, B, world, rank)
    ms, issue = timed(step, feed, _triple(1000 + rank), args.steps, group)
    extra = sum(a.nbytes for a in engine._peer.allocs.values()) if engine._peer else 0
    out = {"device_ms_per_step": round(ms, 3), "samples_per_s": round(world * B * 1e3 / ms, 1),
           "host_issue_ms_per_step": round(issue, 3), "peak_mem_gb": round(peak_gb(extra, group), 2),
           "last_losses": step.losses()}
    release(engine)
    del model, engine, step, feed
    torch.cuda.empty_cache()
    return out


def alone(args, precision, B, T, group):
    """Every rank builds and replays the step alone; -> (its result or None if some rank ran
    out of memory, error text).  Nothing waits on a peer before the OOM flags are exchanged."""
    import torch.distributed as dist
    res, err = None, ""
    try:
        res = run_one(args, precision, B, T, "single", 1, 0, None)
    except torch.cuda.OutOfMemoryError as exc:          # reported, not raised
        err = str(exc).splitlines()[0]
    torch.cuda.empty_cache()
    ok = torch.tensor([0 if err else 1], device="cuda")
    if group is not None:
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
    if not int(ok):
        return None, err or "out of memory on another rank"
    return res, ""


def worker(args):
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    group = None
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        group = dist.group.WORLD
    try:
        for name in args.workloads.split(","):
            B, T, precisions = WORKLOADS[name]
            for precision in precisions:
                head = {"workload": name, "precision": precision, "B_per_gpu": B, "T": T,
                        "n_gpus": world}
                res, err = alone(args, precision, B, T, group)
                if res is None:
                    if rank == 0:
                        print("RESULT " + json.dumps(dict(head, mode="all", oom=True,
                                                          error=err)), flush=True)
                    continue
                if world == 1:
                    print("RESULT " + json.dumps(dict(head, mode="single", **res)), flush=True)
                    continue
                for mode in ["peer", "nccl"] * args.reps:
                    res = run_one(args, precision, B, T, mode, world, rank, group)
                    if rank == 0:
                        print("RESULT " + json.dumps(dict(head, mode=mode, **res)), flush=True)
    finally:
        if group is not None:
            dist.barrier()
            dist.destroy_process_group()


def sweep(args):
    from batch_time import corpus
    from distortion_banks import build_banks
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    have = torch.cuda.device_count()
    ns = [int(n) for n in args.gpus.split(",")]
    run = [n for n in ns if n <= have]
    print(json.dumps({"device": q.splitlines(), "gpus_on_node": have,
                      "not_measured_n": [n for n in ns if n > have]}), flush=True)
    Bmax = max(B for B, _, _ in WORKLOADS.values())
    results = []
    with tempfile.TemporaryDirectory() as root:
        # every rank needs at least two batches per epoch at the largest batch
        data_root, cfg, cache = corpus(root, max(160, 2 * Bmax * max(run)))
        json.dump(build_banks(os.path.join(root, "banks")), open(os.path.join(root, "banks.json"),
                                                                 "w"))
        for n in run:
            cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone",
                   "--nproc_per_node=%d" % n, os.path.abspath(__file__), "--worker",
                   "--root", root, "--data-root", data_root, "--cfg", cfg, "--cache", cache,
                   "--steps", str(args.steps), "--reps", str(args.reps),
                   "--workloads", args.workloads]
            p = subprocess.run(cmd, capture_output=True, text=True)
            lines = [json.loads(l[7:]) for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if p.returncode != 0:
                print(json.dumps({"n_gpus": n, "exit_code": p.returncode,
                                  "stderr_tail": p.stderr.splitlines()[-20:]}), flush=True)
            results += lines
    base = {}
    for r in results:
        if r["n_gpus"] == 1 and "device_ms_per_step" in r:
            base[(r["workload"], r["precision"])] = r["device_ms_per_step"]
    for r in results:
        b = base.get((r["workload"], r["precision"]))
        if b is not None and "device_ms_per_step" in r:
            r["weak_scaling_efficiency"] = round(b / r["device_ms_per_step"], 4)
        print(json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", default="1,2,4,8", help="process counts to run (those the node has)")
    ap.add_argument("--steps", type=int, default=20, help="steps per timed block")
    ap.add_argument("--reps", type=int, default=2, help="peer / nccl alternations per workload")
    ap.add_argument("--workloads", default="c3,c4")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    for k in ("--root", "--data-root", "--cfg", "--cache"):
        ap.add_argument(k, help=argparse.SUPPRESS)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    (worker if a.worker else sweep)(a)


if __name__ == "__main__":
    main()
