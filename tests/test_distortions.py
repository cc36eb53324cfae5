"""On-device PASE+ distortions (pase_b200/distortions.py, pase_b200/csrc/distort.cu).

CPU: the planner reproduces the reference's draw streams (tests/golden/distortions.pt, made
by make_distortion_golden.py from the unmodified reference), the float64 oracle matches the
reference's outputs, and the host orchestration with emulated kernels matches the oracle.
GPU: the FFT convolution against float64 np.convolve, the whole pipeline against the goldens
and the oracle, untouched samples and guard bands, reproducibility, graph replay, refusals.
"""
import json
import os
import random

import numpy as np
import pytest
import torch

import distortions_oracle as DO
import emul
from distortion_banks import (CASES, FULL_CASES, build_banks, case_cfg, golden_view, make_chunk,
                              raw_banks)
from helpers import GOLDEN
from make_distortion_golden import Recorder
from pase_b200 import ops
from pase_b200.distortions import config_distortions

SENT = 1.0e30


@pytest.fixture(scope="module")
def banks(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("distortion_banks"))
    paths = build_banks(root)
    return paths, raw_banks(paths)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "distortions.pt"))


def _meta(golden, name):
    return json.loads(golden[name + "/meta"])


def _seeded_plan(dist, B, T, seed):
    random.seed(seed)
    np.random.seed(seed)
    with Recorder() as rec:
        plan = dist.plan(B, T)
    return plan, rec.log


def _raw_for(dist, paths, raw):
    """The raw banks in the order the distortion object indexes them."""
    out = dict(raw)
    if dist.ir is not None:
        out["irs"] = [raw["irs"][paths["ir_files"].index(n)] for n in dist.ir.names]
    if dist.bd is not None:
        out["bandrop"] = [raw["bandrop"][paths["fir_files"].index(n)] for n in dist.bd.names]
    return out


def _oracle(x, plan, raw):
    return np.stack([DO.distort(x[b].astype(np.float64), plan.samples[b], raw)
                     for b in range(x.shape[0])])


def _oracle_labels(plan, T, d):
    return np.stack([DO.overlap_label(T, s["overlap"]["shift"], d) if "overlap" in s
                     else np.zeros(T // d) for s in plan.samples])


def _errs(y, ref):
    y, ref = np.asarray(y, np.float64), np.asarray(ref, np.float64)
    out = []
    for b in range(ref.shape[0]):
        rel = np.linalg.norm(y[b] - ref[b]) / max(np.linalg.norm(ref[b]), 1e-30)
        mx = np.abs(y[b] - ref[b]).max() / max(np.abs(ref[b]).max(), 1e-30)
        out.append((rel, mx))
    return max(e[0] for e in out), max(e[1] for e in out)


def _golden_errs(y, golden, name):
    """Errors of y ((B, T)) against the reference output the golden keeps: relative L2 and
    max error over the kept samples (every sample for FULL_CASES), scaled by the row's max |y|,
    and the relative error of each row's L2 norm."""
    y = np.asarray(y, np.float64)
    view = golden_view(torch.from_numpy(y)).numpy()
    ref = golden[name + "/y_view"].double().numpy()
    amax = golden[name + "/y_amax"].double().numpy()
    norm = golden[name + "/y_norm"].double().numpy()
    rel = max(np.linalg.norm(view[b] - ref[b]) / max(np.linalg.norm(ref[b]), 1e-30)
              for b in range(ref.shape[0]))
    mx = max(np.abs(view[b] - ref[b]).max() / max(amax[b], 1e-30) for b in range(ref.shape[0]))
    nrm = float(np.max(np.abs(np.linalg.norm(y, axis=1) - norm) / np.maximum(norm, 1e-30)))
    if name in FULL_CASES:
        r2, m2 = _errs(y, golden[name + "/y"].numpy())
        rel, mx = max(rel, r2), max(mx, m2)
    return rel, mx, nrm


# ---------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize("name", list(CASES))
def test_planner_reproduces_reference_draws(name, banks, golden):
    paths, _ = banks
    cfg, B, T, d, seed = case_cfg(name, paths)
    dist = config_distortions(device="cpu", report=True, **cfg)
    plan, log = _seeded_plan(dist, B, T, seed)
    meta = _meta(golden, name)
    want = [ev for s in meta["streams"] for ev in s]
    assert log == want
    rep = dist.sample_report(plan)
    assert [dict(r) for r in rep] == meta["reports"]


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_outputs(name, banks, golden):
    paths, raw = banks
    cfg, B, T, d, seed = case_cfg(name, paths)
    dist = config_distortions(device="cpu", **cfg)
    plan, _ = _seeded_plan(dist, B, T, seed)
    ref = _oracle(make_chunk(B, T, seed), plan, _raw_for(dist, paths, raw))
    rel, mx, nrm = _golden_errs(ref, golden, name)
    # the reference computes in float32 (scipy convolve, np.dot): ~5e-7 relative at T=48000
    assert rel < 3e-6 and mx < 1e-5 and nrm < 3e-6, (rel, mx, nrm)
    lab = _oracle_labels(plan, T, d).astype(np.float32)
    assert np.array_equal(golden[name + "/overlap"].numpy(), lab)


def test_cases_cover_the_bank_edges(banks):
    """The golden cases draw short and long overlap files, and noise files shorter than,
    equal to and longer than T."""
    paths, _ = banks
    seen_ov, seen_noise = set(), set()
    for name in ("overlap", "overlap_reverb", "noise"):
        cfg, B, T, d, seed = case_cfg(name, paths)
        plan, _ = _seeded_plan(config_distortions(device="cpu", **cfg), B, T, seed)
        for s in plan.samples:
            if "overlap" in s:
                seen_ov.add((name, s["overlap"]["file"]))
            if "noise" in s:
                seen_noise.add(s["noise"]["file"])
    assert {("overlap", 0), ("overlap", 1), ("overlap_reverb", 0),
            ("overlap_reverb", 1)} <= seen_ov
    assert seen_noise == {0, 1, 2}


@pytest.mark.parametrize("name", ["reverb_4097", "overlap_reverb", "noise", "clip", "bandrop",
                                  "downsample", "pase_plus"])
def test_emulated_pipeline_matches_oracle(name, banks, monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    paths, raw = banks
    cfg, B, T, d, seed = case_cfg(name, paths)
    dist = config_distortions(device="cpu", **cfg)
    plan, _ = _seeded_plan(dist, B, T, seed)
    x = torch.from_numpy(make_chunk(B, T, seed)).view(B, 1, T)
    x0 = x.clone()
    y, lab = dist.apply(x, plan, torch.zeros(B, 1, T // d))
    assert torch.equal(x, x0)
    rel, mx = _errs(y.view(B, T).numpy(), _oracle(x0.view(B, T).numpy(), plan, _raw_for(dist, paths, raw)))
    assert rel < 1e-6 and mx < 1e-6, (rel, mx)
    assert lab.shape == (B, 1, T // d)
    assert np.array_equal(lab.view(B, -1).numpy(), _oracle_labels(plan, T, d).astype(np.float32))


def test_call_writes_chunk_and_overlap(banks, monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    paths, _ = banks
    cfg, B, T, d, seed = case_cfg("overlap", paths)
    dist = config_distortions(device="cpu", **cfg)
    x = torch.from_numpy(make_chunk(B, T, seed)).view(B, 1, T)
    batch = {"chunk": x, "cchunk": x, "overlap": torch.zeros(B, T // d)}
    out = dist(batch)
    assert out is batch and batch["cchunk"] is x and batch["chunk"] is not x
    assert batch["overlap"].shape == (B, T // d) and float(batch["overlap"].sum()) > 0


@pytest.mark.parametrize("kw,dep", [({}, "codec2_p"),
                                    ({"codec2_p": 0, "chop_factors": [[0.05, 0.025]]}, "chop_p"),
                                    ({"codec2_p": 0, "speed_range": [-0.1, 0.1]}, "speed_p"),
                                    ({"codec2_p": 0, "resample_factors": [4]}, "resample_p")])
def test_unsupported_stages_raise(kw, dep):
    with pytest.raises(NotImplementedError, match=dep):
        config_distortions(device="cpu", **kw)


def test_disabled_stages_draw_nothing(banks):
    paths, _ = banks
    cfg = case_cfg("clip", paths)[0]
    assert config_distortions(device="cpu", **dict(cfg, clip_p=0.0)) is None
    dist = config_distortions(device="cpu", **cfg)
    plan, log = _seeded_plan(dist, 5, 4000, 3)
    assert [ev[0] for ev in log] == ["random", "choice"] * 5
    assert all(set(s) == {"clip"} for s in plan.samples)


def test_empty_file_lists_glob_the_data_root(banks):
    paths, _ = banks
    cfg = dict(case_cfg("bandrop", paths)[0], bandrop_irfiles=[])
    dist = config_distortions(device="cpu", **cfg)
    assert sorted(dist.bd.names) == sorted(paths["fir_files"])
    cfg = dict(case_cfg("reverb_24000", paths)[0], reverb_irfiles=[])
    dist = config_distortions(device="cpu", **cfg)
    assert sorted(dist.ir.names) == sorted(paths["ir_files"])


def test_planner_validates_against_the_banks(banks):
    paths, _ = banks
    cfg = case_cfg("overlap", paths)[0]
    dist = config_distortions(device="cpu", **cfg)
    with pytest.raises(ValueError, match="shift"):
        dist._pack(1, 16000, [{"overlap": {"shift": 16000, "file": 0, "beg": 0, "snr": 5}}])
    with pytest.raises(ValueError, match="segment"):
        dist._pack(1, 16000, [{"overlap": {"shift": 0, "file": 1, "beg": 10 ** 6, "snr": 5}}])


# ---------------------------------------------------------------------------------- GPU

TOL_REL, TOL_MAX = 3e-6, 1e-5


def _conv_ws(B, T, L):
    import ctypes
    from pase_b200 import _lib
    n = ctypes.c_long(0)
    _lib.call("pase_fft_conv_workspace", B, T, L, ctypes.addressof(n))
    return torch.empty((n.value + 15) // 16 * 4, dtype=torch.float32, device="cuda")


def _twiddle():
    from pase_b200.distortions import _twiddles
    return torch.from_numpy(_twiddles()).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("T", [4001, 16000, 32000, 48000])
@pytest.mark.parametrize("L", [1, 101, 103, 4096, 4097, 7000, 24000])
def test_fft_conv_against_numpy(L, T):
    from pase_b200 import _lib
    rng = np.random.RandomState(L * 7 + T)
    # rows: full length, two variable-length segments (overlap Ts = T - s), one not drawn
    ns = [T, T - int(0.75 * T) + 1, T // 2 + 3, T]
    B, ld = len(ns), T + 40
    x = rng.randn(B, T).astype(np.float32)
    h = rng.randn(L).astype(np.float32)
    slack = 64
    bank = torch.full((L + 2 * slack,), SENT, dtype=torch.float32)
    bank[slack:slack + L] = torch.from_numpy(h)
    bank = bank.cuda()
    ps = [0, L // 2, L - 1, L // 3]
    jobs = torch.tensor([[1 if b < 3 else 0, ns[b], slack, L, ps[b], 2] for b in range(B)],
                        dtype=torch.int64).cuda()
    xin = torch.full((B, ld), SENT, dtype=torch.float32)
    xin[:, :T] = torch.from_numpy(x)
    for b in range(B):
        xin[b, ns[b]:T] = SENT               # samples past n must not be read
    xin = xin.cuda()
    out = torch.full((B, ld), -7.0, dtype=torch.float32, device="cuda")
    ws = _conv_ws(B, T, L)
    _lib.call("pase_fft_conv", xin, ld, bank, bank.numel(), jobs, B, T, L, _twiddle(), ws,
              ws.numel() * 4, out, ld)
    o = out.cpu().numpy()
    for b in range(B):
        n = ns[b]
        if b == 3:
            assert (o[b] == -7.0).all()
            continue
        ref = np.convolve(x[b, :n].astype(np.float64), h.astype(np.float64))[ps[b]:ps[b] + n]
        rel = np.linalg.norm(o[b, :n] - ref) / np.linalg.norm(ref)
        mx = np.abs(o[b, :n] - ref).max() / np.abs(ref).max()
        assert rel <= TOL_REL and mx <= TOL_MAX, (b, n, rel, mx)
        assert (o[b, n:] == -7.0).all()                # guard band and tail untouched
    assert torch.equal(bank[:slack].cpu(), torch.full((slack,), SENT))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_fft_conv_energy_modes(mode):
    """FIR (mode 0) and reverb (mode 1) scaling, in place, against the oracle stages."""
    from pase_b200 import _lib
    rng = np.random.RandomState(5 + mode)
    B, T = 3, 16000
    L = 101 if mode == 0 else 7000
    h = rng.randn(L) * np.exp(-np.arange(L) / (L / 5.0))
    h[10] = 5.0
    hn = h / abs(h.max())
    p = int(round(L / 2)) if mode == 0 else int(np.argmax(np.abs(hn)))
    x = rng.randn(B, T).astype(np.float32)
    x[2] = 0.0                                            # zero energy: x (mode 0) / y (mode 1)
    xd = torch.from_numpy(x).cuda()
    bank = torch.from_numpy(hn.astype(np.float32)).cuda()
    jobs = torch.tensor([[1, T, 0, L, p, mode]] * B, dtype=torch.int64).cuda()
    ws = _conv_ws(B, T, L)
    _lib.call("pase_fft_conv", xd, T, bank, L, jobs, B, T, L, _twiddle(), ws, ws.numel() * 4,
              xd, T)
    hf = hn.astype(np.float32).astype(np.float64)
    for b in range(2):
        ref = DO.fir(x[b].astype(np.float64), hf) if mode == 0 else \
            DO.reverb(x[b].astype(np.float64), hf)
        rel, mx = _errs(xd[b:b + 1].cpu().numpy(), ref[None])
        assert rel <= TOL_REL and mx <= TOL_MAX, (b, rel, mx)
    assert (xd[2] == 0).all()


def _gpu_case(name, paths):
    cfg, B, T, d, seed = case_cfg(name, paths)
    return config_distortions(device="cuda", **cfg), B, T, d, seed


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_pipeline_matches_golden_and_oracle(name, banks, golden):
    paths, raw = banks
    dist, B, T, d, seed = _gpu_case(name, paths)
    plan, _ = _seeded_plan(dist, B, T, seed)
    x = torch.from_numpy(make_chunk(B, T, seed)).view(B, 1, T).cuda()
    x0 = x.clone()
    y, lab = dist.apply(x, plan, torch.zeros(B, 1, T // d, device="cuda"))
    assert torch.equal(x, x0)
    y = y.view(B, T).cpu().numpy()
    ref = _oracle(x0.view(B, T).cpu().numpy(), plan, _raw_for(dist, paths, raw))
    rel, mx = _errs(y, ref)
    assert rel <= TOL_REL and mx <= TOL_MAX, ("oracle", rel, mx)
    rel, mx, nrm = _golden_errs(y, golden, name)
    assert rel <= TOL_REL and mx <= TOL_MAX and nrm <= TOL_REL, ("golden", rel, mx, nrm)
    assert torch.equal(lab.view(B, -1).cpu(), golden[name + "/overlap"])


@pytest.mark.gpu
def test_pase_plus_b64_t48000(banks):
    paths, raw = banks
    cfg = case_cfg("pase_plus", paths)[0]
    dist = config_distortions(device="cuda", **cfg)
    B, T, d = 64, 48000, 160
    plan, _ = _seeded_plan(dist, B, T, 99)
    x = torch.from_numpy(make_chunk(B, T, 99)).view(B, 1, T).cuda()
    y, lab = dist.apply(x, plan, torch.zeros(B, T // d, device="cuda"))
    rel, mx = _errs(y.view(B, T).cpu().numpy(), _oracle(x.view(B, T).cpu().numpy(), plan, _raw_for(dist, paths, raw)))
    assert rel <= TOL_REL and mx <= TOL_MAX, (rel, mx)
    assert np.array_equal(lab.cpu().numpy(), _oracle_labels(plan, T, d).astype(np.float32))
    # samples no stage drew come back bit-identical
    idle = [b for b, s in enumerate(plan.samples) if not s]
    assert idle and torch.equal(y.view(B, T)[idle], x.view(B, T)[idle])
    # two runs: equal bits
    y2, lab2 = dist.apply(x, plan, torch.zeros(B, T // d, device="cuda"))
    assert torch.equal(y, y2) and torch.equal(lab, lab2)


@pytest.mark.gpu
def test_all_stages_off_is_identity(banks):
    paths, _ = banks
    dist, B, T, d, seed = _gpu_case("all_48000", paths)
    plan = dist._pack(B, T, [{}] * B)
    x = torch.from_numpy(make_chunk(B, T, seed)).view(B, 1, T).cuda()
    y, lab = dist.apply(x, plan, torch.ones(B, 1, T // d, device="cuda"))
    assert torch.equal(y, x) and not bool(lab.any())


@pytest.mark.gpu
def test_graph_replay_with_new_plan(banks):
    paths, _ = banks
    cfg = case_cfg("pase_plus", paths)[0]
    cfg.update(reverb_p=0.8, overlap_p=0.5, noises_p=0.6, bandrop_p=0.5, downsample_p=0.5)
    dist = config_distortions(device="cuda", **cfg)
    B, T, d = 16, 16000, 160
    x = torch.from_numpy(make_chunk(B, T, 7)).cuda()
    p1, _ = _seeded_plan(dist, B, T, 1)
    p2, _ = _seeded_plan(dist, B, T, 2)
    assert p1.samples != p2.samples
    table = dist.upload(p1)
    y = torch.empty_like(x)
    lab = torch.empty(B, T // d, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                   # warm-up outside the capture
        y.copy_(x)
        dist.run(y, table, p1.offsets, lab, d)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y.copy_(x)
        dist.run(y, table, p1.offsets, lab, d)
    dist.upload(p2, out=table)
    g.replay()
    torch.cuda.synchronize()
    y_ref, lab_ref = dist.apply(x, p2, torch.zeros(B, T // d, device="cuda"))
    assert torch.equal(y, y_ref) and torch.equal(lab, lab_ref)


@pytest.mark.gpu
def test_bad_arguments_are_refused():
    from pase_b200 import _lib
    B, T, L = 2, 1000, 10
    x = torch.zeros(B, T, device="cuda")
    bank = torch.zeros(L, device="cuda")
    jobs = torch.zeros(B, 6, dtype=torch.int64, device="cuda")
    tw = _twiddle()
    ws = _conv_ws(B, T, L)
    nb = ws.numel() * 4
    good = [x, T, bank, L, jobs, B, T, L, tw, ws, nb, x, T]
    _lib.call("pase_fft_conv", *good)
    bad = [(0, None, "x is NULL"), (2, None, "bank is NULL"), (4, None, "jobs is NULL"),
           (8, None, "twiddle is NULL"), (9, None, "ws is NULL"), (11, None, "out is NULL"),
           (1, T - 1, "ldx"), (12, T - 1, "ldo"), (5, 0, "njobs"), (6, 0, "T="),
           (7, 0, "Lmax"), (10, nb - 1, "ws_bytes"), (3, 0, "bank_len")]
    for i, v, msg in bad:
        args = list(good)
        args[i] = v
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("pase_fft_conv", *args)
    mix = torch.zeros(B, 3, dtype=torch.int64, device="cuda")
    snr = torch.ones(B, dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="seg is NULL"):
        _lib.call("pase_noise_mix", x, T, None, T, mix, snr, B, T)
    with pytest.raises(RuntimeError, match="lds"):
        _lib.call("pase_noise_mix", x, T, x, T - 1, mix, snr, B, T)
    with pytest.raises(RuntimeError, match="pool_len"):
        _lib.call("pase_segment_gather", bank, 0, mix, B, T, x, T)
    with pytest.raises(RuntimeError, match="cf is NULL"):
        _lib.call("pase_clip", x, T, jobs, None, B, T)
    lab = torch.zeros(B, T, device="cuda")
    with pytest.raises(RuntimeError, match="does not divide"):
        _lib.call("pase_overlap_label", mix, B, T, 3, lab, T)
    with pytest.raises(RuntimeError, match="ldl"):
        _lib.call("pase_overlap_label", mix, B, T, 10, lab, T // 10 - 1)
