#!/usr/bin/env python
"""Headline benchmark: waveform-samples/sec, PASE+ encoder forward+backward,
(B=32, T=32000) per GPU, fp32 (BASELINE.json metric / configs[1]).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # CPU arm: the reference algorithm (oracle port)

One JSON line on rank 0 (contract in the task description).  A "step" is one pass of the
hot path over one synthetic batch: forward, backward, (N>1: one flat-gradient NCCL
all-reduce), fused Adam update.  `value` = device-timed throughput with inputs resident
in HBM; `e2e` = the same through the public API with pinned HOST waveforms (H2D inside
the timed region) and a D2H read of the loss every step.
"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

PASE_PLUS = {"kwidths": [251, 20, 11, 11, 11, 11, 11, 11], "strides": [1, 10, 2, 1, 2, 1, 2, 2],
             "fmaps": [64, 64, 128, 128, 256, 256, 512, 512], "rnn_dim": 512, "denseskips": True,
             "norm_out": True, "rnn_pool": True, "rnn_layers": 1}
B_PER_GPU, T_CHUNK = 32, 32000
DP_SPLIT = 3          # blocks below this index form the late (small) all-reduce bucket
METRIC = "waveform-samples/sec PASE+ encoder fwd+bwd (B=32,T=32000 per GPU)"
# SURVEY.md 8(d): algorithmic work per 32000-sample chunk
FLOP_PER_CHUNK = 25.4e9          # fwd+bwd as the reference computes it
BYTES_PER_CHUNK = 96.5e6         # ideal-fusion HBM traffic, fp32
FP32_FFMA_PEAK_TF = 67.0         # H100 SXM data sheet: 132 SM x 128 lanes x 2 x 1.98 GHz


def load_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        d = json.load(open(path))
        return {"hbm_gbs": d["hbm_gbs"], "tf": d["bf16_tflops"],
                "tf_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]), "src": "measured"}
    # H100 SXM data sheet (700 W card): HBM3 bandwidth, dense bf16
    return {"hbm_gbs": 3350.0, "tf": 989.0, "tf_sustained": 989.0, "src": "H100 SXM data sheet"}


class ClockSampler(threading.Thread):
    """nvidia-smi style clock / throttle-reason sampling during the timed region (NVML)."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self.reasons, self.stop_flag = index, [], set(), False
        self.max_mhz = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def run(self):
        if self.nv is None:
            return
        nv = self.nv
        names = {
            getattr(nv, "nvmlClocksThrottleReasonSwPowerCap", 0x4): "sw_power_cap",
            getattr(nv, "nvmlClocksThrottleReasonHwSlowdown", 0x8): "hw_slowdown",
            getattr(nv, "nvmlClocksThrottleReasonSwThermalSlowdown", 0x20): "sw_thermal_slowdown",
            getattr(nv, "nvmlClocksThrottleReasonHwThermalSlowdown", 0x40): "hw_thermal_slowdown",
            getattr(nv, "nvmlClocksThrottleReasonHwPowerBrakeSlowdown", 0x80): "hw_power_brake",
        }
        while not self.stop_flag:
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                mask = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                for bit, nm in names.items():
                    if mask & bit:
                        self.reasons.add(nm)
            except Exception:
                pass
            time.sleep(0.05)

    def summary(self):
        s = sorted(self.samples)
        med = s[len(s) // 2] if s else None
        return {"sm_mhz": med, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(s)}


def physical_gpu_index(local):
    vis = os.environ.get("CUDA_VISIBLE_DEVICES")
    if vis:
        try:
            return int(vis.split(",")[local])
        except Exception:
            return local
    return local


# ------------------------------------------------------------------ CPU arm ---
def oracle_step_fn(batch):
    """fwd+bwd+Adam of the reference algorithm (CPU oracle port) on `batch` chunks."""
    import pase_oracle as O
    from pase_b200.frontend import WaveFe
    torch.manual_seed(0)
    sd = WaveFe(**PASE_PLUS).state_dict()           # reference default initialisation
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()
              if v.is_floating_point() and "running" not in k}
    full = dict(sd)
    full.update(leaves)
    opt = torch.optim.Adam(list(leaves.values()), lr=1e-4)
    x = torch.randn(batch, 1, T_CHUNK)

    def step():
        opt.zero_grad(set_to_none=True)
        y = O.encoder_forward(x, full, PASE_PLUS, training=True, new_stats={})
        loss = y.square().mean()
        loss.backward()
        opt.step()
        return float(loss.detach())
    return step


def usable_cores():
    """Host cores this process may actually use: scheduler affinity capped by the cgroup
    CPU quota (a container that reports 128 CPUs but is throttled to a few would otherwise
    oversubscribe torch's thread pool and crawl)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q = open("/sys/fs/cgroup/cpu.max").read().split()
        if q[0] != "max":
            n = min(n, max(1, int(float(q[0]) / float(q[1]))))
    except Exception:
        try:
            quota = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if quota > 0:
                n = min(n, max(1, quota // period))
        except Exception:
            pass
    return max(1, n)


def time_cpu(batch, steps, warmup, budget_s=None):
    cores = usable_cores()
    # torch's intra-op pool stops scaling on this conv stack well before 64 threads
    torch.set_num_threads(min(cores, 64))
    step = oracle_step_fn(batch)
    for _ in range(warmup):
        step()
    ts = []
    t_begin = time.perf_counter()
    for _ in range(steps):
        t0 = time.perf_counter()
        step()
        ts.append(time.perf_counter() - t0)
        if budget_s is not None and time.perf_counter() - t_begin > budget_s:
            break
    steps = len(ts)
    total = sum(ts)
    return {"value": batch * T_CHUNK * steps / total, "sec_per_step": total / steps,
            "min_sec": min(ts), "cores": torch.get_num_threads(), "batch": batch, "steps": steps}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    # the SAME configuration as the native arm: one step = the full B=32 batch (a few seconds
    # of CPU work); the 200 s budget only cuts the number of timed steps on a slow host
    batch = B_PER_GPU
    r = time_cpu(batch, args.steps, min(args.warmup, 3), budget_s=200.0)
    args.steps = r["steps"]          # fewer than asked only if the budget ran out
    line = {
        "impl": "reference", "metric": METRIC, "value": r["value"], "unit": "samples/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": min(args.warmup, 3),
        "ms_per_step": r["sec_per_step"] * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "PASE+.cfg encoder fwd+bwd+adam, T=32000, fp32, train-mode BN, "
                               "no workers (BASELINE configs[1])",
                   "global_batch": batch, "seq_len": T_CHUNK, "parallelism": "cpu-threads"},
        "cpu_baseline": {"value": r["value"], "unit": "samples/s", "cores": r["cores"],
                         "kind": "port",
                         "sample": "the full B=%d batch of 32000-sample chunks per step; "
                                   "reference algorithm via oracle/pase_oracle.py (torch CPU "
                                   "ops, QRNN as python scan: torchqrnn is un-vendored, parity "
                                   "for that layer unpinned)" % batch},
        "e2e": {"value": r["value"], "unit": "samples/s", "h2d_bytes_per_step": 0,
                "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def workers_plus_cfg():
    """cfg/workers/workers+.cfg restated programmatically (names, output sizes, r, losses)."""
    mlp = lambda name, nout: {"num_outputs": nout, "dropout": 0, "hidden_size": 256,
                              "hidden_layers": 1, "name": name, "context": 1, "r": 7,
                              "loss": "MSELoss", "skip": False}
    regr = [{"num_outputs": 1, "dropout": 0, "dropout_time": 0.0, "hidden_layers": 1,
             "name": "cchunk", "type": "decoder", "hidden_size": 64, "fmaps": [512, 256, 128],
             "strides": [4, 4, 10], "kwidths": [30, 30, 30], "loss": "L1Loss"}]
    for name, nout in (("lps", 3075), ("lps_long", 3075), ("fbank", 120), ("fbank_long", 120),
                       ("gtn", 120), ("gtn_long", 120), ("mfcc", 39), ("mfcc_long", 60),
                       ("prosody", 12)):
        regr.append(mlp(name, nout))
    cls = [{"num_outputs": 1, "dropout": 0, "hidden_size": 256, "hidden_layers": 1, "name": n,
            "loss": "BCEWithLogitsLoss", "skip": False, "augment": n == "cmi"}
           for n in ("mi", "cmi")]
    return {"regr": regr, "cls": cls}


def time_workers(dev, precision, B, T=T_CHUNK, steps=5, warmup=3, graph=True, stream=None,
                 fuse=True):
    """BASELINE configs[2]/[3] shape on one GPU: PASE+ encoder on the 3B concatenated chunks +
    all 12 workers+ heads + summed loss, fwd + bwd + ONE flat Adam launch; the whole step
    replayed as one CUDA graph when `graph`.  -> dict (ms/step, chunk-samples/s, ...)."""
    from pase_b200.pase import pase, total_loss
    from pase_b200.utils import parse_workers
    from pase_b200 import functional as Fn
    from pase_b200.optim import FlatAdam
    Fn.set_precision(precision)
    torch.manual_seed(0)
    wcfg = workers_plus_cfg()
    model = pase(frontend_cfg=dict(PASE_PLUS), minions_cfg=parse_workers(wcfg)).to(dev).train()
    model.frontend.precision = precision
    # fused output layer + contextualised MSE for the MLP regression heads (3xF16): the
    # (B, F*r, T') predictions -- 551 MB each for the two lps heads -- are never stored
    model.fuse_regression_loss = (precision == "3xf16") and fuse
    Tq = T // 160
    batch = {k: torch.randn(B, 1, T, device=dev) for k in
             ("chunk", "chunk_ctxt", "chunk_rand", "cchunk")}
    for w in wcfg["regr"]:
        if w["name"] != "cchunk":
            batch[w["name"]] = torch.randn(B, w["num_outputs"], Tq, device=dev)
    # the reference steps 13 Adam instances (trainer.py:86-143); here: one launch
    opt = FlatAdam([p for p in model.parameters()], lr=1e-4).bind_encoder(model.frontend)
    loss_dev = torch.zeros((), device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        h, chunk, preds, labels = model(batch, 1, dev)
        tot, _ = total_loss(model, preds, labels)
        tot.backward()
        opt.step()
        loss_dev.copy_(tot.detach())
    stream = stream or torch.cuda.current_stream()
    with torch.cuda.stream(stream):
        for _ in range(max(warmup, 3)):
            step()
    stream.synchronize()
    fn, graphed, why = step, False, None
    if graph:
        try:
            opt.zero_grad(set_to_none=True)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                step()
            fn, graphed = g.replay, True
            for _ in range(2):
                fn()
        except Exception as exc:
            why = repr(exc)[:200]
            torch.cuda.synchronize()
    ms = _event_time(fn, steps)
    nparam = sum(p.numel() for p in model.parameters())
    # algorithmic FLOPs of the step as the reference computes it (SURVEY.md 8d, per step at
    # B=32: encoder on the 3B = 96 chunks 2438 GFLOP, 9 MLP heads 487, cchunk decoder 1409),
    # scaled with B; counted once per product whatever the GEMM mode issues
    gflop = (2438.0 + 487.0 + 1409.0) * B / 32.0 * (T / float(T_CHUNK))
    pk = load_peaks()
    peak = pk["tf_sustained"]
    ach = gflop / ms                      # GFLOP / ms = TFLOP/s
    roof = {"bound": "tensor", "achieved": ach, "peak": peak, "unit": "TFLOP/s",
            "frac": ach / peak, "traffic": None,
            "algorithmic_gflop_per_step": gflop,
            "note": "FLOPs as the reference computes the step (SURVEY.md 8d), counted once per "
                    "product; peak = bf16 tensor rate (" + pk["src"] + ")"}
    return {"metric": "waveform-samples/sec PASE+ encoder(3B chunks)+workers+ heads fwd+bwd+adam",
            "roofline": roof,
            "value": B * T / (ms * 1e-3), "unit": "chunk-samples/s", "ms_per_step": ms,
            "n_gpus": 1, "cuda_graph": graphed, "graph_error": why,
            "loss": float(loss_dev),
            "config": {"workload": "PASE+.cfg + workers+.cfg (12 workers), B=%d chunk triplets, "
                                   "T=%d" % (B, T),
                       "gemm_precision": precision, "params": nparam,
                       "fused_regression_heads": bool(model.fuse_regression_loss),
                       "optimizer": "pase_adam_flat, one launch for all 13 parameter groups"},
            "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}


def run_workers(args):
    """Extra workload (BASELINE configs[2-3] shape).  Not the contract line."""
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    side = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(side)
    print(json.dumps(time_workers(dev, args.precision, args.batch, steps=args.steps,
                                  warmup=args.warmup, graph=not args.no_graph, stream=side,
                                  fuse=not args.no_fuse_heads)),
          flush=True)


# ------------------------------------------------------------------ extra legs ---
def _event_time(fn, steps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def measure_matmul_peaks(dev):
    """Dense tensor-core peaks of THIS GPU as cuBLAS reaches them (torch.matmul, 8192^3, best
    of 5 bursts of 10 back-to-back GEMMs): TF32, fp16 and bf16.  Denominators for the
    issued-MMA fractions."""
    out = {}
    n = 8192
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        for name, dt, tf32 in (("tf32", torch.float32, True), ("fp16", torch.float16, False),
                               ("bf16", torch.bfloat16, False)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            a = torch.randn(n, n, device=dev, dtype=dt)
            b = torch.randn(n, n, device=dev, dtype=dt)
            for _ in range(3):
                a @ b
            best = min(_event_time(lambda: a @ b, 10) for _ in range(5))
            out[name + "_tflops"] = 2.0 * n ** 3 / (best * 1e-3) / 1e12
            del a, b
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def library_baseline(dev, steps=5):
    """SURVEY 8(d) / BASELINE.md 4.4: the reference's own module graph on this GPU through
    the vendor libraries (cuDNN conv / batch-norm, cuBLAS), `cudnn.benchmark=True` as
    train.py:26 sets it: the oracle restatement with lib_ops on CUDA tensors, fwd + bwd +
    fused Adam on the same synthetic (32,1,32000) batch, once with TF32 allowed (PyTorch's
    cuDNN default) and once strict fp32.  QRNN: python scan over 200 frames (torchqrnn's
    runtime-compiled kernel is un-vendored)."""
    import pase_oracle as O
    from pase_b200.frontend import WaveFe
    torch.manual_seed(0)
    sd = {k: v.to(dev) for k, v in WaveFe(**PASE_PLUS).state_dict().items()}
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()
              if v.is_floating_point() and "running" not in k}
    full = dict(sd)
    full.update(leaves)
    opt = torch.optim.Adam(list(leaves.values()), lr=1e-4, fused=True)
    x = torch.randn(B_PER_GPU, 1, T_CHUNK, device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        y = O.encoder_forward(x, full, PASE_PLUS, training=True, new_stats={}, lib_ops=True)
        y.square().mean().backward()
        opt.step()
    res = {}
    prev = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
            torch.backends.cuda.matmul.allow_tf32)
    try:
        torch.backends.cudnn.benchmark = True
        for name, allow in (("tf32_allowed", True), ("fp32_strict", False)):
            torch.backends.cudnn.allow_tf32 = allow
            torch.backends.cuda.matmul.allow_tf32 = allow
            for _ in range(3):
                step()
            ms = _event_time(step, steps)
            res[name] = {"ms_per_step": ms, "value": B_PER_GPU * T_CHUNK / (ms * 1e-3)}
    finally:
        (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
         torch.backends.cuda.matmul.allow_tf32) = prev
    res["what"] = ("oracle/pase_oracle.py encoder_forward(lib_ops=True) on CUDA: F.conv1d / "
                   "F.batch_norm / F.prelu (cuDNN, cuBLAS), cudnn.benchmark=True, eager, fused "
                   "Adam; B=32, T=32000")
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    return res


def time_encoder_config(dev, stream, precision, B, T, steps=10):
    """ms/step of the native encoder fwd+bwd+Adam at another (precision, B, T) operating
    point, whole step replayed as one CUDA graph (inputs resident)."""
    from pase_b200 import wf_builder
    from pase_b200.graph import GraphedEncoderStep
    torch.manual_seed(0)
    model = wf_builder(dict(PASE_PLUS)).to(dev).train()
    model.precision = precision
    from pase_b200.optim import FlatAdam
    opt = FlatAdam(list(model.parameters()), lr=1e-4).bind_encoder(model)
    gs = GraphedEncoderStep(model, opt, lambda y: y.square().mean(), (B, 1, T), dev,
                            stream=stream, resident=True,
                            x_init=torch.randn(B, 1, T))
    for _ in range(3):
        gs.step()
    ms = _event_time(gs.step, steps)
    mem = sum(p.nbytes() for p in model._plans.values()) / 2 ** 30
    del gs, opt, model
    torch.cuda.empty_cache()
    return {"precision": precision, "batch": B, "seq_len": T, "ms_per_step": ms,
            "value": B * T / (ms * 1e-3), "unit": "samples/s", "plan_gb": mem}


def gemm_time_in_replay(step_fn, gemm_flop_per_step, peak_tflops, reps=3):
    """Sum of the tensor-core GEMM kernels' device durations inside `reps` replays of the
    captured step, from torch.profiler's CUDA activity records."""
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            step_fn()
        torch.cuda.synchronize()
    us, n = 0.0, 0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "tc_gemm" in e.name:
            us += e.time_range.end - e.time_range.start
            n += 1
    if n == 0:
        raise RuntimeError("no GEMM kernel records")
    ms = us / 1e3 / reps
    ach = gemm_flop_per_step / (ms * 1e-3) / 1e12
    return {"gemm_ms_per_step": ms, "gemm_launches_per_step": n // reps, "achieved": ach,
            "unit": "TFLOP/s", "frac": ach / peak_tflops,
            "how": "torch.profiler CUDA activity records of %d graph replays" % reps}


def time_lps_targets(dev, B=B_PER_GPU, T=T_CHUNK, reps=10):
    """SURVEY.md 8f N1: the lps + lps_long regression targets of one step computed ON the GPU
    from the chunks already resident there (pase_b200/targets.py), next to the reference's way
    (torch.stft + librosa-style deltas per chunk on the host, then an H2D copy of the labels)."""
    import time
    from pase_b200.targets import LPS
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import targets_oracle as TO
    wav = torch.randn(B, 1, T, device=dev) * 0.3
    tr = [LPS(win=400, name="lps"), LPS(win=512, name="lps_long")]
    for t in tr:
        t(wav)
    ms = _event_time(lambda: [t(wav) for t in tr], reps)
    w0 = wav[0, 0].cpu()
    t0 = time.perf_counter()
    n_cpu = 2
    for _ in range(n_cpu):
        TO.lps(w0, 2048, 160, 400, 2)
        TO.lps(w0, 2048, 160, 512, 2)
    cpu_ms_chunk = (time.perf_counter() - t0) / n_cpu * 1e3
    nbytes = 2 * B * 3075 * (T // 160) * 4
    return {"config": "N1: lps + lps_long regression targets of one step on the GPU, B=%d, "
                      "T=%d (2 x (B, 3075, %d) fp32)" % (B, T, T // 160),
            "ms_per_step": ms, "launches": 6,
            "label_bytes_not_copied_h2d": nbytes,
            "cpu_reference_ms_per_chunk": cpu_ms_chunk,
            "cpu_reference_ms_per_step_one_core": cpu_ms_chunk * B,
            "note": "reference path = oracle/targets_oracle.py (torch.stft + savgol deltas) per "
                    "chunk on one host core, as a DataLoader worker runs it"}


def dump_outputs(d, arrays):
    """arrays: name -> tensor (float32 / float64), written as d/<name>.npy"""
    import numpy as np
    os.makedirs(d, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(d, name + ".npy"), t.cpu().numpy())


# ------------------------------------------------------------------ GPU arm ---
def run_native(args):
    import torch.distributed as dist
    from pase_b200 import wf_builder, ops
    from pase_b200.dp import FlatGradAllReducer

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run for --gpus > 1")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    # everything runs on one non-default stream so that the eager steps and the CUDA-graph
    # capture of the end-to-end step share their autograd (AccumulateGrad) stream
    side = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(side)

    torch.manual_seed(0)                               # identical replicas
    model = wf_builder(dict(PASE_PLUS)).to(dev).train()
    model.precision = args.precision
    params = list(model.parameters())
    # ONE flat fp32 gradient buffer: the encoder's backward kernels write their gradients
    # straight into it (WaveFe.grad_sink), N>1 all-reduces it with one NCCL call, and one
    # pase_adam_flat launch updates every parameter (pase_b200/optim.py).
    # --torch-adam: the round-1 path (autograd-accumulated gradients packed into a flat
    # buffer, ATen fused Adam) for A/B comparison.
    from pase_b200.optim import FlatAdam
    red = None
    peer = False
    if args.torch_adam:
        red = FlatGradAllReducer(params, attach=False) if world > 1 else None
        opt = torch.optim.Adam(params, lr=1e-4, fused=True)
        grad_bytes = red.nbytes if red is not None else 0
    else:
        n_lower = None
        if world > 1 and args.overlap:
            # flat buffer ordered [blocks 0..2 | rest]: the all-reduce of the large bucket is
            # hidden behind the backward of blocks 2..0 (pase_b200/graph.py::PipelinedDPStep)
            from pase_b200.graph import PipelinedDPStep
            params, n_lower = PipelinedDPStep.order_params(model, DP_SPLIT)
        if world > 1 and args.dp == "peer" and not args.overlap:
            # data parallelism fused into the update: peer-mapped flat buffers, ONE kernel does
            # the gradient mean over this rank's shard, Adam and the parameter all-gather over
            # NVLink (pase_adam_flat_dp) -- no collective call, the step stays one CUDA graph
            try:
                opt = FlatAdam(params, lr=1e-4, peer_dp=True).bind_encoder(model)
                peer = True
            except Exception as exc:          # noqa: BLE001 -- every rank fails together
                sys.stderr.write("bench: peer-mapped DP unavailable (%s); NCCL all-reduce\n" % (exc,))
        if not peer:
            opt = FlatAdam(params, lr=1e-4).bind_encoder(model)
        grad_bytes = opt.n * 4 if world > 1 else 0

    def zero_grads():
        opt.zero_grad(set_to_none=True)

    def reduce_grads():
        if red is not None:
            red.pack_and_reduce()
        elif world > 1:
            opt.reduce_grads()
    g = torch.Generator(device="cpu").manual_seed(1000 + rank)   # distinct data per rank
    x_host = torch.randn(B_PER_GPU, 1, T_CHUNK, generator=g).pin_memory()
    x_dev = x_host.to(dev)

    last = {}

    def loss_of(y):
        """the step's loss; keeps the step's output and loss for --dump-outputs (in a captured
        step these are the graph's static tensors, rewritten by every replay)"""
        last["output"] = y
        last["loss"] = y.square().mean()
        return last["loss"]

    def step_resident():
        zero_grads()
        y = model(x_dev)
        loss = loss_of(y)
        loss.backward()
        reduce_grads()
        opt.step()
        return loss

    def step_e2e():
        zero_grads()
        y = model(x_host, device=dev)                   # H2D of the pinned waveform batch
        loss = y.square().mean()
        loss.backward()
        reduce_grads()
        opt.step()
        return loss.item()                              # D2H read of the step's result

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    for _ in range(max(args.warmup, 3)):
        step_resident()
    # launches of OUR kernels per step, counted on eager steps (a graph replay re-issues the
    # same kernels without going through the Python funnel)
    n0 = ops.launch_count
    step_resident()
    launches_per_step = ops.launch_count - n0
    value_fn, value_graphed = step_resident, False
    gopt = gres = gs = None
    # N>1: two captured halves ([fwd, bwd, pack gradients] and [Adam]) with the NCCL
    # all-reduce of the flat gradient buffer issued eagerly between the two replays
    if world > 1 and not (not args.torch_adam and peer):
        gkw = dict(post_backward=red.pack, between=red.reduce) if red is not None else \
            dict(between=opt.reduce_grads)
    else:
        gkw = {}
    if not args.no_graph:
        try:
            from pase_b200.graph import GraphedEncoderStep
            gopt = torch.optim.Adam(params, lr=1e-4, fused=True, capturable=True) \
                if args.torch_adam else opt
            if world > 1 and not args.torch_adam and args.overlap:
                gres = PipelinedDPStep(model, opt, loss_of,
                                       (B_PER_GPU, 1, T_CHUNK), dev, split=DP_SPLIT,
                                       n_lower=n_lower, stream=side, resident=True)
            else:
                gres = GraphedEncoderStep(model, gopt, loss_of,
                                          (B_PER_GPU, 1, T_CHUNK), dev, stream=side,
                                          resident=True, **gkw)
            gres.x_static.copy_(x_dev)
            value_fn, value_graphed = (lambda: gres.step()), True
            for _ in range(3):
                value_fn()
        except Exception as exc:
            sys.stderr.write("bench: CUDA-graph capture unavailable (%s); eager steps\n" % (exc,))
    sampler = ClockSampler(physical_gpu_index(local)) if rank == 0 else None
    if sampler:
        sampler.start()
    ms = timed(value_fn, args.steps)
    launches = launches_per_step * args.steps
    if sampler:
        sampler.stop_flag = True
        sampler.join(timeout=2)
    if args.dump_outputs and rank == 0:
        # what the last timed step returned: its loss and encoder output, and the parameters
        # its Adam update wrote (7.8 M fp32), before any later step touches them
        dump_outputs(args.dump_outputs, {
            "loss": last["loss"].detach().double(),
            "output": last["output"].detach().float(),
            "params": torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])})

    # end-to-end: through the public API with pinned HOST waveforms; the whole step (H2D, fwd,
    # bwd, Adam, D2H of the loss) is captured in one CUDA graph (N>1: two, around the
    # all-reduce) when possible
    graphed, e2e_fn = False, step_e2e
    if not args.no_graph:
        try:
            from pase_b200.graph import GraphedEncoderStep
            gopt = gopt or (torch.optim.Adam(params, lr=1e-4, fused=True, capturable=True)
                            if args.torch_adam else opt)
            if world > 1 and not args.torch_adam and args.overlap:
                gs = PipelinedDPStep(model, opt, lambda y: y.square().mean(),
                                     (B_PER_GPU, 1, T_CHUNK), dev, split=DP_SPLIT,
                                     n_lower=n_lower, stream=side)
            else:
                gs = GraphedEncoderStep(model, gopt, lambda y: y.square().mean(),
                                        (B_PER_GPU, 1, T_CHUNK), dev, stream=side,
                                        prefetch=not args.no_prefetch, **gkw)
            gs.x_host.copy_(x_host)                   # the loader's pinned staging buffer
            e2e_fn = lambda: gs.step()
            graphed = True
        except Exception as exc:                      # report, fall back to the eager path
            sys.stderr.write("bench: CUDA-graph capture unavailable (%s); eager e2e\n" % (exc,))
    for _ in range(2):
        e2e_fn()
    ms_e2e = timed(e2e_fn, args.steps)

    samples_per_step = B_PER_GPU * T_CHUNK * world
    value = samples_per_step * args.steps / (ms * 1e-3)
    e2e_value = samples_per_step * args.steps / (ms_e2e * 1e-3)

    # ---- roofline of the dominant kernel family (implicit-GEMM): CUDA events around each
    # gemm launch of one extra, untimed-for-the-headline step -------------------------------
    gemm_ms, gemm_flop, per_kernel = 0.0, 0.0, {}
    recs = []
    real_call = ops.call

    def spy(name, *a):
        if name in ("pase_gemm_nt", "pase_gemm_tn", "pase_tc_gemm_nt", "pase_tc_gemm_tn"):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = real_call(name, *a)
            e.record()
            if name == "pase_gemm_nt":
                fl = 2.0 * a[6] * a[7] * a[8]
            elif name == "pase_gemm_tn":
                fl = 2.0 * a[10] * a[11] * a[12] * a[13]
            elif name == "pase_tc_gemm_nt":
                fl = 2.0 * a[9] * a[10] * a[11]
            else:
                fl = 2.0 * a[12] * a[13] * a[14] * a[15]
            recs.append((name, s, e, fl))
            return r
        return real_call(name, *a)
    # every rank runs the two instrumented steps (they contain the gradient all-reduce, a
    # collective); only rank 0 records
    if rank == 0:
        ops.call = spy
    try:
        for _ in range(2):
            recs.clear()
            step_resident()
            torch.cuda.synchronize()
    finally:
        ops.call = real_call
    for name, s, e, fl in recs:
        t = s.elapsed_time(e)
        gemm_ms += t
        gemm_flop += fl
        k = per_kernel.setdefault(name, [0, 0.0, 0.0])
        k[0] += 1
        k[1] += t
        k[2] += fl
    if world > 1:
        dist.barrier()

    if rank == 0:
        peaks = load_peaks()
        step_ms = ms / args.steps
        ach_tf = gemm_flop / (gemm_ms * 1e-3) / 1e12 if gemm_ms > 0 else 0.0
        chunks = B_PER_GPU
        hbm_ach = BYTES_PER_CHUNK * chunks / (step_ms * 1e-3) / 1e9
        line = {
            "metric": METRIC, "value": value, "unit": "samples/s", "n_gpus": world,
            "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": step_ms,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": {"fp32": "f32", "3xtf32": "f32 (3xTF32 split on wgmma, fp32 accumulate: "
                      "fp32-equivalent products)",
                      "3xf16": "f32 (3xF16 split on wgmma, fp32 accumulate: fp32-equivalent "
                               "products)", "tf32": "tf32", "bf16": "bf16"}[args.precision],
            "data": "synthetic",
            "parity": "oracle pinned to goldens of the unmodified reference (tests/golden); the "
                      "QRNN layer follows SURVEY.md A.2 (torchqrnn is un-vendored and unpinned "
                      "upstream: parity for that layer is unpinned)",
            "config": {"workload": "PASE+.cfg encoder fwd+bwd+adam, B=32/GPU, T=32000, fp32, "
                                   "train-mode BN, no workers (BASELINE configs[1])",
                       "global_batch": B_PER_GPU * world, "seq_len": T_CHUNK,
                       "parallelism": "dp%d" % world, "gemm_precision": args.precision,
                       "cuda_graph": value_graphed,
                       "l2": "no flush: per-step working set (~1.7 GB activations) >> 50 MB L2",
                       "optimizer": "torch fused Adam" if args.torch_adam else
                       ("pase_adam_flat_dp (one launch, moments sharded over the ranks)"
                        if peer else "pase_adam_flat (one launch, gradients written in place)"),
                       "grad_allreduce": None if world == 1 else (
                           "one flat buffer; upper bucket overlapped with backward of blocks "
                           "%d..0 (side stream), lower bucket after" % (DP_SPLIT - 1)
                           if (args.overlap and not args.torch_adam) else
                           ("fused into the update kernel over peer memory (pase_adam_flat_dp: "
                            "mean of the peers' gradient shards + Adam + parameter all-gather "
                            "over NVLink, no collective call, one CUDA graph per step)"
                            if (not args.torch_adam and peer) else
                            "one ncclAllReduce(avg) of the flat buffer between two graph replays")),
                       "grad_allreduce_bytes": grad_bytes},
            "e2e": {"value": e2e_value, "unit": "samples/s", "ms_per_step": ms_e2e / args.steps,
                    "cuda_graph": graphed, "input_prefetch": bool(graphed and not args.no_prefetch),
                    "h2d_bytes_per_step": x_host.numel() * 4, "d2h_bytes_per_step": 4},
            "gpu_launches": launches,
            "clocks": sampler.summary() if sampler else None,
            "roofline": {
                "kernel": {"fp32": "pase_gemm_nt + pase_gemm_tn (fp32 FFMA implicit-GEMM conv "
                                   "fwd/dgrad/wgrad)",
                           "3xtf32": "pase_tc_gemm_nt + pase_tc_gemm_tn (wgmma tf32, 3 MMAs "
                                     "per product; FLOPs counted once)",
                           "3xf16": "pase_tc_gemm_nt + pase_tc_gemm_tn (wgmma f16 on fp16 "
                                    "hi/lo pairs, 3 MMAs per product; FLOPs counted once)",
                           "bf16": "pase_tc_gemm_nt + pase_tc_gemm_tn (wgmma bf16)",
                           "tf32": "pase_tc_gemm_nt + pase_tc_gemm_tn (wgmma tf32)"}[
                    args.precision],
                "bound": "tensor", "achieved": ach_tf, "peak": peaks["tf_sustained"],
                "unit": "TFLOP/s", "frac": ach_tf / peaks["tf_sustained"],
                "peak_source": peaks["src"] + " bf16",
                "gemm_share_of_step": gemm_ms / step_ms if step_ms > 0 else None,
                "gemm_ms_per_step": gemm_ms, "gemm_gflop_per_step": gemm_flop / 1e9,
                "frac_of_fp32_ffma_peak": ach_tf / FP32_FFMA_PEAK_TF,
                "per_kernel": {k: {"launches": v[0], "ms": v[1], "tflops": v[2] / (v[1] * 1e-3) / 1e12
                                   if v[1] > 0 else 0.0} for k, v in per_kernel.items()},
                "step_hbm": {"algorithmic_bytes_per_step": BYTES_PER_CHUNK * chunks,
                             "achieved_gbs": hbm_ach, "peak_gbs": peaks["hbm_gbs"],
                             "frac": hbm_ach / peaks["hbm_gbs"]},
                "step_flops": {"algorithmic_flop_per_step": FLOP_PER_CHUNK * chunks,
                               "achieved_tflops": FLOP_PER_CHUNK * chunks / (step_ms * 1e-3) / 1e12},
            },
        }
        if world == 1 and not args.no_extras:
            # everything below is measured AFTER the timed regions of the headline numbers
            gs = None                       # release the e2e graph's memory pool
            torch.cuda.empty_cache()
            pk = measure_matmul_peaks(dev)
            line["peaks_measured_here"] = pk
            issued = {"3xtf32": (3.0, "tf32_tflops"), "tf32": (1.0, "tf32_tflops"),
                      "3xf16": (3.0, "fp16_tflops"), "bf16": (1.0, "bf16_tflops")}.get(args.precision)
            if issued:
                line["roofline"]["issued_mma_tflops"] = issued[0] * ach_tf
                line["roofline"]["issued_mma_frac_of_pipe_peak"] = issued[0] * ach_tf / pk[issued[1]]
                line["roofline"]["pipe_peak"] = "%s dense, torch.matmul 8192^3 on this GPU: %.0f " \
                    "TFLOP/s" % (issued[1].split("_")[0], pk[issued[1]])
            try:
                line["library_baseline"] = library_baseline(dev)
            except Exception as exc:                      # never lose the headline line
                line["library_baseline"] = {"error": repr(exc)[:300]}
            others = []
            for (prec, B, T, tag) in (
                    ("bf16", B_PER_GPU, T_CHUNK, "BASELINE configs[2] encoder part: bf16, B=32, T=32000"),
                    ("bf16", 64, 48000, "BASELINE configs[4] shape: bf16, B=64/GPU, T=48000"),
                    ("3xtf32", B_PER_GPU, T_CHUNK, "previous default numerics (round 1)")):
                if prec == args.precision and B == B_PER_GPU and T == T_CHUNK:
                    continue
                try:
                    r = time_encoder_config(dev, side, prec, B, T)
                    r["config"] = tag
                    others.append(r)
                except Exception as exc:
                    others.append({"config": tag, "error": repr(exc)[:300]})
            try:
                w = time_workers(dev, args.precision, B_PER_GPU, stream=side)
                w["config"]["baseline"] = "BASELINE configs[2]/[3] per-GPU shape"
                others.append(w)
            except Exception as exc:
                others.append({"config": "workers+ full step", "error": repr(exc)[:300]})
            try:
                others.append(time_lps_targets(dev))
            except Exception as exc:
                others.append({"config": "on-device lps targets", "error": repr(exc)[:300]})
            line["other_configs"] = others
            if value_graphed and gres is not None:
                # LAST (profiling must not touch any timed number): the GEMM launches' device
                # time INSIDE the graph replay that `value` times (CUPTI activity records through
                # torch.profiler: no per-launch events, no launch gaps, warm caches), next to
                # the event-bracketed figure of `roofline.achieved`
                try:
                    line["roofline"]["in_replay"] = gemm_time_in_replay(
                        lambda: gres.step(), gemm_flop, peaks["tf_sustained"])
                except Exception as exc:                  # never lose the headline line
                    line["roofline"]["in_replay"] = {"error": repr(exc)[:200]}
            gres = None
        if world == 1 and not args.no_cpu_baseline:
            r = time_cpu(4, 3, 1, budget_s=30.0)
            line["cpu_baseline"] = {
                "value": r["value"], "unit": "samples/s", "cores": r["cores"], "kind": "port",
                "sec_per_step": r["sec_per_step"],
                "sample": "4 chunks x 32000 samples, <=3 timed fwd+bwd+adam iterations (30 s "
                          "budget) of the reference algorithm (oracle/pase_oracle.py) on the "
                          "host cores"}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dp", default="peer", choices=["peer", "nccl"],
                    help="N>1 gradient exchange: 'peer' = fused into the update kernel over "
                         "CUDA-IPC peer memory (pase_adam_flat_dp: reduce-scatter + Adam + "
                         "all-gather, one CUDA graph per step, no collective call); 'nccl' = one "
                         "ncclAllReduce(avg) of the flat buffer between two graph replays")
    ap.add_argument("--overlap", action="store_true",
                    help="N>1: hide the all-reduce of the large gradient bucket behind the tail "
                         "of backward (PipelinedDPStep, three graphs + side stream); the extra "
                         "graph launches, events and SM contention can cost more than the "
                         "all-reduce of 31 MB over NVLink, so the plain form is the default")
    ap.add_argument("--no-fuse-heads", action="store_true",
                    help="workers workload: materialise the regression predictions (reference "
                         "protocol) instead of fusing output layer + contextualised MSE")
    ap.add_argument("--no-prefetch", action="store_true",
                    help="e2e: copy the step's batch H2D inside the step instead of prefetching "
                         "the next batch on a copy stream during the current step")
    ap.add_argument("--torch-adam", action="store_true",
                    help="round-1 optimizer path (ATen fused Adam on autograd-accumulated grads)")
    ap.add_argument("--no-extras", action="store_true",
                    help="skip the legs measured after the headline: cuBLAS pipe peaks, the "
                         "cuDNN library baseline, the other operating points")
    ap.add_argument("--no-graph", action="store_true", help="eager end-to-end step (no CUDA graph)")
    ap.add_argument("--workload", default="encoder", choices=["encoder", "workers"],
                    help="encoder = the contract line (BASELINE configs[1]); workers = encoder + "
                         "all workers+ heads (informational)")
    ap.add_argument("--batch", type=int, default=32, help="chunk triplets per step (workers workload)")
    ap.add_argument("--precision", default=os.environ.get("PASE_B200_PRECISION", "3xf16"),
                    choices=["fp32", "3xtf32", "3xf16", "tf32", "bf16"],
                    help="GEMM numerics: fp32 FFMA; 3xTF32 / 3xF16 wgmma (fp32-equivalent); TF32 "
                         "wgmma; bf16 wgmma with bf16 activation storage (BASELINE configs[2,4])")
    ap.add_argument("--dump-outputs", metavar="DIR",
                    help="encoder workload: after the timed steps, write the last timed step's "
                         "loss, encoder output and updated parameters as DIR/<name>.npy")
    args = ap.parse_args()
    if args.dump_outputs and (args.impl != "native" or args.workload != "encoder"):
        raise SystemExit("--dump-outputs: encoder workload of the native implementation only")
    if args.impl == "reference":
        run_reference(args)
    elif args.workload == "workers":
        run_workers(args)
    else:
        run_native(args)


if __name__ == "__main__":
    main()
