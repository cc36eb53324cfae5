"""WaveFe.extract_long / FeatureStream (windowed inference of one long recording) on the GPU:
bit-equal to the whole-recording forward in every precision, against the float64 oracle, the
select_output modes, a recording beyond the packed forward's 32-bit limit in bounded memory,
streaming against extract_long, and argument errors raised before any launch."""
import random

import pytest
import torch

import pase_oracle as O
import pase_b200.ops as ops
from pase_b200 import _lib
from pase_b200 import encoder as enc
from helpers import resolve_cfg, fill_state_dict, seeded_randn, assert_close
from pase_b200.frontend import WaveFe

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "3xtf32", "3xf16", "bf16"]
CFGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
SEED = 11
W = 81920                                     # the minimum window: 512 frames


def _model(cfg_name, precision="3xf16"):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.load_state_dict(fill_state_dict(m.state_dict(), SEED))
    m.precision = precision
    return m.cuda().eval()


def _whole(m, x, mode=None):
    with torch.no_grad():
        return m(x.view(1, 1, -1).cuda(), mode=mode)


def test_window_minimum_is_the_sequential_scan():
    assert _lib.qrnn_scan_plan(enc.MIN_WINDOW_FRAMES) != 0
    assert _lib.qrnn_scan_plan(enc.MIN_WINDOW_FRAMES + 1) == 0


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg_name", CFGS)
def test_extract_long_bit_equal_to_whole(cfg_name, precision):
    m = _model(cfg_name, precision)
    for i, (L, window) in enumerate([(4 * W + 160 * 31, W), (3 * W + 160 * 200 + 1, W + 160 * 5),
                                     (6 * W + 160 * 17 + 150, 160 * 517)]):
        x = seeded_randn((L,), 40 + i, 0.5)
        assert len(enc.plan_windows(m.cfg, L, window)) >= 3
        got = m.extract_long(x if i % 2 else x.cuda(), window=window)
        y = _whole(m, x)
        assert got.is_cuda and got.shape == y.shape
        assert torch.equal(got, y), "L=%d window=%d: max |diff| %.3g" % (
            L, window, float((got - y).abs().max()))


def test_extract_long_unwindowable_lengths():
    m = _model("cfg/frontend/PASE+.cfg")
    before = ops.launch_count
    with pytest.raises(NotImplementedError, match="pools its dense skips"):
        m.extract_long(torch.zeros(3 * W + 159), window=W)
    assert ops.launch_count == before
    p = _model("cfg/frontend/PASE.cfg")                       # no dense skips: any length
    x = seeded_randn((3 * W + 159,), 9, 0.5)
    assert torch.equal(p.extract_long(x, window=W), _whole(p, x))


def test_extract_long_matches_oracle_3xf16():
    cfg = resolve_cfg("cfg/frontend/PASE+.cfg")
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    sd = fill_state_dict(WaveFe(**cfg).state_dict(), SEED)
    x = seeded_randn((300000,), 77, 0.5)
    got = m.extract_long(x, window=W)
    with torch.no_grad():
        ref = O.encoder_forward(x.view(1, 1, -1), sd, cfg, training=False)
    assert_close(got, ref, 1e-3, 1e-5, "oracle")


def test_extract_long_modes():
    m = _model("cfg/frontend/PASE+.cfg")
    x = seeded_randn((3 * W + 1234,), 5, 0.5)
    h = m.extract_long(x, window=W)
    for mode in ("avg_norm", "avg_concat", "avg_norm_concat"):
        g = m.extract_long(x, mode=mode, window=W)
        ref = O.select_output(h.cpu(), mode)
        assert g.shape == ref.shape
        assert float((g.cpu() - ref).abs().max()) <= 1e-6 * float(h.abs().max()), mode


def test_extract_long_beyond_the_packed_limit():
    m = _model("cfg/frontend/PASE+.cfg", "bf16")
    L = 40_000_000
    x = seeded_randn((L,), 123, 0.5)
    with pytest.raises(ValueError, match="32-bit"):
        m.extract([x])
    outs, stats = [], []
    for window in (1 << 20, 3 * W):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        y = m.extract_long(x, window=window)
        torch.cuda.synchronize()
        plan = m._packed_plans[next(reversed(m._packed_plans))]
        peak = torch.cuda.max_memory_allocated() - base
        out_bytes = y.numel() * 4
        # the window plan (allocated in this call), the output, and 64 MB for the GEMM operand
        # conversions and the allocator's rounding
        assert peak <= plan.nbytes() + out_bytes + (64 << 20), (window, peak, plan.nbytes())
        outs.append(y.cpu())
        del y
    assert torch.equal(outs[0], outs[1])
    # allocations after warm-up: the output only, whatever the number of windows
    counts = []
    for L2 in (5 * W + 160 * 3, 9 * W + 160 * 7):
        x2 = seeded_randn((L2,), L2, 0.5)
        torch.cuda.synchronize()
        n0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        y = m.extract_long(x2, window=3 * W)
        torch.cuda.synchronize()
        counts.append(torch.cuda.memory_stats()["allocation.all.allocated"] - n0)
        del y
    assert counts == [1, 1], counts


def test_stream_matches_extract_long():
    m = _model("cfg/frontend/PASE+.cfg")
    cfg = m.cfg
    L = W + 160 * 100 + 77
    x = seeded_randn((L,), 31, 0.5)
    ref = m.extract_long(x, window=W)
    assert torch.equal(ref, _whole(m, x))
    rng = random.Random(7)
    for size in (160, 1000, 48000, None, 1):             # None: random sizes
        st = m.stream()
        outs, a = [], 0
        while a < L:
            n = size if size is not None else rng.randrange(1, 30000)
            if size == 1 and a < L - 3000:
                n = rng.randrange(1, 4000)           # single samples over the last 3000 only
            y = st.push(x[a:a + n] if size != 48000 else x[a:a + n].cuda())
            a = min(a + n, L)
            assert y.shape[2] == enc.final_frames(cfg, a) - sum(o.shape[2] for o in outs)
            outs.append(y)
        outs.append(st.finish())
        got = torch.cat(outs, 2)
        assert torch.equal(got, ref), (size, float((got - ref).abs().max()))


def test_stream_latency_rule():
    cfg = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    _, B = enc.receptive_field(cfg)
    n = 10 * W + 160 * 37 + 12
    f = enc.final_frames(cfg, n)
    assert 160 * (f - 1) + B <= n - 1 < 160 * f + B


def test_argument_errors_before_any_launch():
    m = _model("cfg/frontend/PASE+.cfg")
    before = ops.launch_count
    with pytest.raises(ValueError, match="window"):
        m.extract_long(torch.zeros(3 * W), window=W - 160)
    with pytest.raises(ValueError, match="recording"):
        m.extract_long(torch.zeros(2, 3 * W))
    with pytest.raises(ValueError, match="mode"):
        m.stream(mode="avg_norm")
    with pytest.raises(ValueError, match="window"):
        m.stream(window=1000)
    m.train()
    with pytest.raises(RuntimeError, match="eval"):
        m.extract_long(torch.zeros(3 * W))
    cpu = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg")).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        cpu.extract_long(torch.zeros(3 * W))
    assert ops.launch_count == before
