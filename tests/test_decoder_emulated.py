"""The cchunk decoder's host logic (geometry, padded-row plan, polyphase weight layout, crop
offsets, row maps of the three GEMMs) on the CPU, with the kernels emulated (tests/emul/):
end to end against float64 conv_transpose1d + PReLU, and stage by stage through the checks and
bounds of tests/test_decoder_gpu.py, at the geometries that file runs on the GPU."""
import pytest
import torch
import torch.nn.functional as F

import emul
import pase_b200.ops as ops
from pase_b200 import functional as Fn
from pase_b200.decoder import decoder_stack, _LayerGeom
from pase_b200.minions import DecoderMinion
from test_decoder_gpu import EDGES, WPLUS, decoder_case, deconv_params, make_minion, \
    poly_weight, _within

CASES = dict(EDGES)
CASES["workers+"] = (256, WPLUS["fmaps"], WPLUS["strides"], WPLUS["kwidths"], 2, 3)


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    monkeypatch.setattr(Fn, "PRECISION", Fn.PRECISION)       # restored after the test


def _reference(m, x, B, T):
    """float64 conv_transpose1d + PReLU from the same fp32 parameters: output (B, L, C) and
    autograd leaves."""
    leaves = [t.detach().double().requires_grad_(True) for trio in deconv_params(m) for t in trio]
    xr = x.detach().double().requires_grad_(True)
    h = xr.view(B, T, -1).permute(0, 2, 1)
    for i, blk in enumerate(m.blocks[:m.n_deconv]):
        W, b, a = leaves[3 * i:3 * i + 3]
        h = F.prelu(F.conv_transpose1d(h, W, b, stride=blk.stride, padding=blk.pad), a)
    return h.permute(0, 2, 1), xr, leaves


@pytest.mark.parametrize("prec", ["fp32", "3xtf32", "3xf16"])
@pytest.mark.parametrize("case", list(CASES))
def test_decoder_against_conv_transpose(case, prec, emulated):
    """Output, input gradient and every weight, bias and slope gradient within 2e-5 of the
    largest float64 value of that tensor (the emulation rounds each GEMM once to fp32)."""
    Fn.set_precision(prec)
    Cin, fm, st, kw, B, T = CASES[case]
    m = make_minion(Cin, fm, st, kw, "cpu", seed=7)
    x = torch.randn(B * T, Cin, generator=torch.Generator().manual_seed(7)).requires_grad_(True)
    out, L = decoder_stack(m, x, B, T)
    ref, xr, leaves = _reference(m, x, B, T)
    assert tuple(ref.shape) == (B, L, fm[-1])
    G = torch.randn(ref.shape, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    out.backward(G.float().reshape(B * L, -1))
    (ref * G.float().double()).sum().backward()
    got = [out.view(B, L, -1), x.grad] + [t.grad for trio in deconv_params(m) for t in trio]
    want = [ref, xr.grad] + [t.grad for t in leaves]
    names = ["out", "dx"] + ["%s%d" % (n, i) for i in range(len(fm)) for n in ("dW", "db", "da")]
    for n, a, b in zip(names, got, want):
        b = b.detach()
        _within(n, a, b, 2e-5 * float(b.abs().max()))


@pytest.mark.parametrize("prec", ["fp32", "3xtf32", "3xf16", "tf32", "bf16"])
@pytest.mark.parametrize("case", ["workers+", "k<s", "k%s==0", "T_in=1", "ffma-96"])
def test_stage_checks_hold_for_emulation(case, prec, emulated):
    """The GPU file's stage checks and bounds, on the emulated kernels (which round each GEMM
    once): every check runs and passes."""
    Cin, fm, st, kw, B, T = CASES[case]
    m = make_minion(Cin, fm, st, kw, "cpu", seed=9)
    res = decoder_case(m, B, T, "cpu", prec, seed=9)
    assert len(res) >= 7 * len(fm) and all(r <= 1.0 for _, r in res)


def test_bounds_are_not_vacuous():
    got = torch.tensor([1.0, 2.0, 3.0])
    ref = got.double()
    tol = torch.tensor([1e-7, 2e-7, 0.0], dtype=torch.float64)
    _within("ok", got, ref, tol)
    for i, d in ((0, 2e-7), (1, 4e-7), (2, 2.0 ** -22)):
        bumped = got.double().clone()
        bumped[i] += d
        with pytest.raises(AssertionError, match="out of bound"):
            _within("bumped", bumped, ref, tol)


def test_poly_weight_is_conv_transpose():
    """The float64 polyphase reference of the GPU file is ConvTranspose1d (padding 0)."""
    for (Cin, Cout, k, s, T) in ((5, 3, 30, 4, 6), (4, 2, 2, 4, 3), (3, 2, 9, 3, 1), (2, 3, 5, 5, 4)):
        gen = torch.Generator().manual_seed(k * s)
        W = torch.randn(Cin, Cout, k, generator=gen, dtype=torch.float64)
        x = torch.randn(2, Cin, T, generator=gen, dtype=torch.float64)
        g = _LayerGeom(Cin, Cout, k, s, 0, T)
        xp = torch.zeros(2, g.Pd, Cin, dtype=torch.float64)
        xp[:, g.taps - 1:g.taps - 1 + T] = x.permute(0, 2, 1)
        X = torch.as_strided(xp, (2, g.U, g.taps * Cin), (g.Pd * Cin, Cin, 1))
        y = (X @ poly_weight(W, s, g.taps).view(s * Cout, -1).t()).view(2, g.U * s, Cout)
        ref = F.conv_transpose1d(x, W, stride=s).permute(0, 2, 1)
        n = ref.shape[1]
        assert torch.allclose(y[:, :n], ref, atol=1e-12) and bool((y[:, n:] == 0).all())


@pytest.mark.parametrize("k,s", [(30, 4), (30, 10), (2, 4), (5, 5), (2, 2), (8, 4), (9, 3),
                                 (3, 5), (1, 1), (31, 3)])
@pytest.mark.parametrize("T", [1, 2, 7, 200])
def test_layer_length_matches_conv_transpose(k, s, T):
    blk = DecoderMinion(4, 1, 0.0, fmaps=[4], strides=[s], kwidths=[k], hidden_size=4).blocks[0]
    g = _LayerGeom(4, 4, k, s, blk.pad, T)
    n = torch.nn.ConvTranspose1d(4, 4, k, stride=s, padding=blk.pad)(torch.zeros(1, 4, T)).shape[2]
    assert g.L == n
    assert g.taps == -(-k // s) and g.U * s >= (T - 1) * s + k


@pytest.mark.parametrize("k,s", [(3, 4), (30, 3), (2, 5), (5, 2)])
def test_mixed_parity_is_refused(k, s):
    """The reference crops one extra sample when k and s differ in parity; not implemented."""
    with pytest.raises(NotImplementedError, match="odd/even"):
        DecoderMinion(64, 1, 0.0, fmaps=[64], strides=[s], kwidths=[k])
