"""WaveFe.extract (packed variable-length inference) on the GPU: every utterance bit-equal to
its own B=1 forward in every precision, against the CPU oracle, the select_output modes,
capacity splitting, launch count and allocations independent of the lengths, and argument
errors raised before any launch."""
import random

import pytest
import torch

import pase_oracle as O
import pase_b200.ops as ops
from helpers import resolve_cfg, fill_state_dict, seeded_randn, assert_close
from pase_b200.frontend import WaveFe

pytestmark = pytest.mark.gpu

LENGTHS = [471, 1000, 1763, 3200, 4001, 12345, 16000, 16001, 31999, 48000, 82081, 100000]
PRECISIONS = ["fp32", "tf32", "3xtf32", "3xf16", "bf16"]
SEED = 11


def _model(cfg_name, precision):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.load_state_dict(fill_state_dict(m.state_dict(), SEED))
    m.precision = precision
    return m.cuda().eval()


def _corpus(lengths, seed=5):
    order = list(lengths) + [1763, 16000, 471]          # duplicates
    random.Random(seed).shuffle(order)
    return [seeded_randn((T,), 100 + i, 0.5) for i, T in enumerate(order)]


def _single(m, w, mode=None):
    with torch.no_grad():
        return m(w.view(1, 1, -1).cuda(), mode=mode)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg_name", ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"])
def test_extract_bit_equal_to_single(cfg_name, precision):
    m = _model(cfg_name, precision)
    wavs = _corpus(LENGTHS)
    feats = m.extract(wavs)                     # CPU inputs, one pack
    assert len(feats) == len(wavs)
    for i, (w, f) in enumerate(zip(wavs, feats)):
        y = _single(m, w)
        assert f.is_cuda and f.shape == y.shape, (i, tuple(f.shape), tuple(y.shape))
        assert torch.equal(f, y), "utterance %d (%d samples): max |diff| %.3g" % (
            i, w.numel(), float((f - y).abs().max()))


def test_extract_matches_oracle_3xf16():
    cfg = resolve_cfg("cfg/frontend/PASE+.cfg")
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    sd = fill_state_dict(WaveFe(**cfg).state_dict(), SEED)
    wavs = [seeded_randn((T,), 7 + T, 0.5) for T in (1763, 16001, 82081)]
    feats = m.extract([w.cuda() for w in wavs])           # CUDA inputs
    for w, f in zip(wavs, feats):
        with torch.no_grad():
            ref = O.encoder_forward(w.view(1, 1, -1), sd, cfg, training=False)
        assert_close(f, ref, 1e-3, 1e-5, "oracle T=%d" % w.numel())


def test_extract_modes():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    wavs = _corpus([471, 3200, 16001, 48000])
    base = m.extract(wavs)
    for mode in ("avg_norm", "avg_concat", "avg_norm_concat"):
        got = m.extract(wavs, mode=mode)
        for i, (h, g) in enumerate(zip(base, got)):
            ref = O.select_output(h.cpu(), mode)
            tol = 1e-6 * float(h.abs().max())
            assert g.shape == ref.shape
            assert float((g.cpu() - ref).abs().max()) <= tol, (mode, i)


def test_extract_capacity_split():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    wavs = _corpus([471, 1000, 3200, 4001, 12345, 31999, 48000])
    cap = 40000                                       # several packs; 48000 exceeds the cap
    feats = m.extract(wavs, max_samples=cap)
    assert len(m._packed_plans) == 2
    for i, (w, f) in enumerate(zip(wavs, feats)):
        assert torch.equal(f, _single(m, w)), i


def test_extract_launches_independent_of_count():
    m = _model("cfg/frontend/PASE+.cfg", "bf16")
    counts = []
    for n in (4, 40):
        wavs = [seeded_randn((2000 + 97 * i,), i, 0.5) for i in range(n)]
        before = ops.launch_count
        m.extract(wavs, mode="avg_norm")
        counts.append(ops.launch_count - before)
    assert counts[0] == counts[1], counts


def test_extract_allocates_nothing_after_warmup():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    m.extract(_corpus([1000, 3200, 16000]))            # warm-up: the packed plan
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    for seed in range(3):
        lengths = random.Random(seed).sample(range(471, 60000), 6)
        wavs = [seeded_randn((T,), T, 0.5) for T in lengths]
        n0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        feats = m.extract(wavs)
        torch.cuda.synchronize()
        # one device allocation per call: the returned features' buffer
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - n0 == 1, seed
        assert len({f.untyped_storage().data_ptr() for f in feats}) == 1
        del feats
        assert torch.cuda.memory_allocated() == base, seed
    assert len(m._packed_plans) == 1


def test_extract_argument_errors():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    before = ops.launch_count
    assert m.extract([]) == []
    with pytest.raises(ValueError, match="utterance 1 .*block"):
        m.extract([torch.zeros(1000), torch.zeros(470)])
    with pytest.raises(ValueError, match="utterance 0"):
        m.extract([torch.zeros(3, 1000)])
    m.train()
    with pytest.raises(RuntimeError, match="eval"):
        m.extract([torch.zeros(1000)])
    cpu = WaveFe(**resolve_cfg("cfg/frontend/PASE+.cfg")).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        cpu.extract([torch.zeros(1000)])
    assert ops.launch_count == before
