"""wgmma / TMA GEMM kernels against the exact spec (the product of the operands as the
tensor core reads them, accumulated in fp64).  Modes 1 (3xTF32) and 3 (3xF16) must be
fp32-equivalent; mode 0 (TF32) and mode 2 (bf16) are exact products of rounded operands, so
they too are checked tightly against the spec evaluated on the SAME rounded operands.

The shape tables reach the kernels' own code paths: the persistent NT loop with several tiles
per CTA, the split weight-gradient GEMM (per-split partial tiles summed in split order) in each
of its regimes, asserted through pase_tc_gemm_tn_plan, and the scalar store path.  Operand
memory the kernels must not use is filled with a huge finite sentinel, so any read of it shows
up as a large error."""
import math

import pytest
import torch

import emul
from pase_b200 import _lib
from test_kernels_gpu import R

pytestmark = pytest.mark.gpu


def _operands(x, mode, weights=False, scale=None):
    """(hi, lo) tensors of operand x in GEMM mode `mode` (CPU)."""
    if mode == 0:
        return x, None
    if mode == 1:
        return _split(x, weights)
    if mode == 2:
        return x.to(torch.bfloat16), None
    v = x if scale is None else x * scale
    hi = v.to(torch.float16)
    return hi, ((v - hi.float()) * 2048.0).to(torch.float16)


def _split(x, weights=False):
    """(hi, lo) as the product builds them: activations pass the raw array as 'hi' (the
    tensor core truncates it) with lo = rn(x - trunc(x)); weights get explicit rn hi/lo."""
    lo = torch.zeros_like(x)
    if weights:
        hi = torch.zeros_like(x)
        emul.core.pase_split_tf32(x, hi, lo, x.numel())
        return hi, lo
    emul.core.pase_split_tf32(x, None, lo, x.numel())
    return x.clone(), lo


def _poison(parts, mask):
    """Fill the operand elements where `mask` is set with a huge finite value: 2^100 in fp32
    and bf16, the largest finite fp16 (65504) in fp16.  Finite, because the kernels multiply
    such reads by TMA zero fill where the contract allows them (0 x finite = 0)."""
    for t in parts:
        if t is not None:
            t[mask[:t.numel()]] = 65504.0 if t.dtype == torch.float16 else 2.0 ** 100


def _run(name, args, offset_args=()):
    """Spec on CPU clones, kernel on device copies.  Arguments listed in `offset_args` are
    passed to both as views starting one element into their buffer (a C that is not 8-byte
    aligned)."""
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    for i in offset_args:
        cpu[i], dev[i] = cpu[i][1:], dev[i][1:]
    emul.call(name, *cpu)
    _lib.call(name, *dev)
    torch.cuda.synchronize()
    return cpu, dev


def test_split_kernel_bit_exact():
    x = R(100003, seed=1) * 37.0
    hi, lo = _split(x, weights=True)
    dh, dl = torch.zeros_like(x).cuda(), torch.zeros_like(x).cuda()
    _lib.call("pase_split_tf32", x.cuda(), dh, dl, x.numel())
    assert torch.equal(dh.cpu(), hi) and torch.equal(dl.cpu(), lo)
    assert float((x - hi - lo).abs().max()) <= float(x.abs().max()) * 2.0 ** -22
    _, lo_a = _split(x)
    dl2 = torch.zeros_like(x).cuda()
    _lib.call("pase_split_tf32", x.cuda(), None, dl2, x.numel())       # activation form
    assert torch.equal(dl2.cpu(), lo_a)
    xt = emul.core._tf32_trunc(x)
    assert float((x - xt - lo_a).abs().max()) <= float(x.abs().max()) * 2.0 ** -21


def _legacy(n, *row):
    """A table row that predates the trailing columns: it keeps its test id, made of its first
    n values, so the case stays comparable across versions of the table."""
    return pytest.param(*row, id="-".join(str(v) for v in row[:n]))


def _nt_tiles(M, N):
    return math.ceil(M / 128) * math.ceil(N / (64 if N <= 64 else 128))


# edge tokens: "ldb" = B rows padded to ldb = K + 8, the padding poisoned; "slackA" = A rows
# past the last row any valid (m, k) reads poisoned; "ldc" = odd ldc (N + 1); "coff" = C one
# element into its buffer (not 8-byte aligned); "multi" = more than 2 x SMs tiles, so every
# CTA of the persistent loop runs at least three tiles (asserted against the device).
NT_CASES = [
    # M, N, K, R, rows_in, t_valid, rows_out, fold, bias, stats, acc, edge
    # one full tile, plain; block-1 like, k spans 2 rows; stride-2 k=11 shape
    _legacy(11, 256, 128, 128, 128, 256, 256, 256, 1, True, True, 0, ""),
    _legacy(11, 1000, 64, 1280, 640, 103, 100, 100, 1, True, True, 0, "slackA"),
    _legacy(11, 700, 128, 704, 128, 70, 64, 64, 1, True, True, 0, "ldb"),
    # two 128-wide column tiles; folded sinc (fold 32); long K, accumulate; dcat shape, wide N
    _legacy(11, 300, 256, 1408, 128, 300, 300, 300, 1, False, False, 0, ""),
    _legacy(11, 520, 2048, 288, 32, 130, 4100, 129, 32, False, True, 0, ""),
    _legacy(11, 333, 512, 5632, 1024, 111, 100, 100, 1, True, False, 1, "ldb"),
    _legacy(11, 260, 1920, 256, 256, 260, 260, 260, 1, False, False, 0, ""),
    # K % 32 != 0: partial k-block; 64 tiles across row groups
    _legacy(11, 300, 128, 200, 64, 300, 300, 300, 1, True, True, 0, ""),
    _legacy(11, 4000, 256, 2816, 256, 1000, 990, 990, 1, True, True, 0, "slackA"),
    (9000, 512, 256, 256, 1000, 990, 990, 1, True, True, 0, "multi slackA"),   # 284 tiles, stats
    (9000, 512, 640, 128, 1000, 990, 990, 1, True, True, 0, "multi ldb"),      # + K > 512 folds
    (700, 100, 256, 256, 700, 700, 700, 1, True, True, 0, ""),          # N tail (emb_dim 100)
    (330, 100, 1280, 640, 110, 100, 100, 1, True, True, 0, "ldc"),      # N tail, odd ldc
    (300, 128, 704, 128, 100, 97, 97, 1, True, True, 0, "ldc coff"),    # scalar store path
    (300, 256, 512, 128, 300, 300, 300, 1, True, True, 0, ""),          # K = 512: one chunk
    (300, 256, 520, 128, 300, 300, 300, 1, True, True, 0, "ldb"),       # last chunk: 1 partial kb
]


@pytest.mark.parametrize("mode", [1, 0, 3, 2])
@pytest.mark.parametrize("M,N,K,Rr,rows_in,t_valid,rows_out,fold,bias,stats,acc,edge", NT_CASES)
def test_tc_gemm_nt(M, N, K, Rr, rows_in, t_valid, rows_out, fold, bias, stats, acc, edge, mode):
    if mode >= 2:
        if Rr % 64 or (K * 2) % 16:
            pytest.skip("16-bit modes need folded rows of 64 elements")
    if "multi" in edge:
        tiles, sms = _nt_tiles(M, N), _lib.device_info()["sms"]
        print("NT %dx%d: %d tiles on %d SMs" % (M, N, tiles, sms))
        assert tiles > 2 * sms, "case no longer reaches the persistent loop's 3rd tile"
    ldb = K + 8 if "ldb" in edge else K
    ldc = N + 1 if "ldc" in edge else N
    a_rows = M + (K + Rr - 1) // Rr + 2
    A = R(a_rows * Rr, seed=11)
    B = R(N * ldb, seed=12, scale=0.1)
    groups = (M + rows_in - 1) // rows_in
    C = R(groups * rows_out * ldc + 8, seed=13)
    bs = R(N, seed=14) if bias else None
    cs = torch.zeros(N, dtype=torch.float64) if stats else None
    cq = torch.zeros(N, dtype=torch.float64) if stats else None
    (Ah, Al), (Bh, Bl) = _operands(A, mode), _operands(B, mode, weights=True)
    if "ldb" in edge:
        _poison((Bh, Bl), (torch.arange(N * ldb) % ldb) >= K)
    if "slackA" in edge:
        _poison((Ah, Al), torch.arange(a_rows * Rr) >= (M + (K - 1) // Rr) * Rr)
    args = [Ah, Al, a_rows, Rr, Bh, Bl, ldb, C, ldc, M, N, K, 0.5, None, bs, rows_in, t_valid,
            rows_out, fold, cs, cq, acc, mode, 0]
    cpu, dev = _run("pase_tc_gemm_nt", args, (7,) if "coff" in edge else ())
    scale = float((A.abs().mean() * B.abs().mean() * K ** 0.5))
    # split modes: fp32-equivalent; single-pass modes: exact products, fp32 accumulation in
    # the tensor core (rounding drift over K)
    tol = (2e-6 if mode in (1, 3) else 2e-5) * max(scale, 1e-3) * 8
    out_c, out_d = cpu[7], dev[7].cpu()
    err = float((out_c - out_d).abs().max())
    assert err <= tol, "C max err %.3e > %.3e (mode %d)" % (err, tol, mode)
    if stats:
        for i in (19, 20):
            c, d = cpu[i].float(), dev[i].cpu().float()
            e = float((c - d).abs().max())
            lim = (2e-5 if mode in (1, 3) else 2e-4) * max(float(c.abs().max()), 1.0)
            assert e <= lim, "stats arg %d err %.3e > %.3e" % (i, e, lim)


@pytest.mark.parametrize("mode", [2, 3, 1])
@pytest.mark.parametrize("M,N,K,Rr,rows_in,t_valid,rows_out,fold,edge", [
    _legacy(8, 1000, 64, 1280, 640, 103, 100, 100, 1, ""),        # BN=64
    _legacy(8, 700, 128, 704, 128, 70, 64, 64, 1, ""),            # BN=128
    _legacy(8, 520, 4096, 320, 64, 130, 8200, 129, 64, ""),  # folded sinc (fold 64), wide N, stats
    _legacy(8, 300, 256, 5632, 1024, 300, 300, 300, 1, ""),       # two column tiles, long K
    (300, 192, 704, 128, 100, 97, 97, 1, "ldc coff"),   # odd ldc, C not 4-byte aligned
    (9000, 512, 256, 256, 1000, 990, 990, 1, "multi"),  # persistent loop, >= 3 tiles per CTA
])
def test_tc_gemm_nt_bf16_out_and_alpha_dev(M, N, K, Rr, rows_in, t_valid, rows_out, fold, edge,
                                           mode):
    """bf16 output (C rounded once from the fp32 result) and the device-side alpha that
    undoes a power-of-two operand scale (3xF16 gradients)."""
    if "multi" in edge:
        assert _nt_tiles(M, N) > 2 * _lib.device_info()["sms"]
    ldc = N + 1 if "ldc" in edge else N
    a_rows = M + (K + Rr - 1) // Rr + 2
    A = R(a_rows * Rr, seed=31) * (1e-6 if mode == 3 else 1.0)     # tiny gradients
    B = R(N * K, seed=32, scale=0.1)
    groups = (M + rows_in - 1) // rows_in
    s = 2.0 ** 32 if mode == 3 else 1.0
    alpha_dev = torch.tensor([1.0 / s, s]) if mode == 3 else None
    (Ah, Al), (Bh, Bl) = _operands(A, mode, scale=s), _operands(B, mode, weights=True)
    cs, cq = torch.zeros(N, dtype=torch.float64), torch.zeros(N, dtype=torch.float64)
    for c16 in ((1, 0) if mode != 1 else (1,)):
        C = torch.zeros(groups * rows_out * ldc + 8, dtype=torch.bfloat16 if c16 else torch.float32)
        args = [Ah, Al, a_rows, Rr, Bh, Bl, K, C, ldc, M, N, K, 1.0, alpha_dev, None, rows_in,
                t_valid, rows_out, fold, cs.clone(), cq.clone(), 0, mode, c16]
        cpu, dev = _run("pase_tc_gemm_nt", args, (7,) if "coff" in edge else ())
        out_c, out_d = cpu[7].float(), dev[7].cpu().float()
        ref_scale = float(out_c.abs().max())
        assert ref_scale > 0
        err = (out_c - out_d).abs()
        if c16:     # one bf16 ulp where the fp32 results straddle a rounding boundary
            assert bool((err <= 2.0 ** -7 * out_c.abs() + 1e-5 * ref_scale).all()), float(err.max())
            assert float((err > 1e-5 * ref_scale).float().mean()) < 0.02
        else:
            assert float(err.max()) <= (2e-5 if mode == 2 else 4e-6) * ref_scale
        for i in (19, 20):      # statistics come from the fp32 values before rounding
            c, d = cpu[i].float(), dev[i].cpu().float()
            assert float((c - d).abs().max()) <= 2e-4 * max(float(c.abs().max()), 1e-30)


# ---- split weight-gradient GEMM ----
# A chunk is one pipeline stage: 32 reduction rows in modes 0/1, 64 in 2/3; a group has
# cpg = ceil(rpg / chunk) chunks; the split modes fold their accumulators every 128 rows
# (flush_ch chunks).  Regime tags, asserted through pase_tc_gemm_tn_plan in every mode the
# case runs in (a tag "t:01" only in modes 0 and 1):
_REGIMES = {
    "one": lambda p: p["splits"] == 1,
    "split": lambda p: p["splits"] > 1,
    "2-8": lambda p: 2 <= p["splits"] <= 8,
    ">16": lambda p: p["splits"] > 16,
    "mid": lambda p: p["splits"] > 1 and p["cps"] % p["cpg"] != 0,      # split inside a group
    "uneven": lambda p: p["splits"] > 1 and p["total"] % p["cps"] != 0,  # short last split
    "unfolded": lambda p: p["splits"] > 1 and p["cps"] % p["flush"] != 0,  # cps % flush_ch
    "unblocked": lambda p: p["splits"] > 1 and p["R"] % p["bn"] != 0,   # b_blocked == 0
    "bn64": lambda p: p["splits"] > 1 and p["bn"] == 64,
    # one more split would exceed the 4 x SMs CTA bound although chains of >= 8 chunks allow it
    "capped": lambda p: p["splits"] > 1 and (p["splits"] + 1) * p["tiles"] > 4 * p["sms"]
    and math.ceil(p["total"] / (p["splits"] + 1)) >= 8,
}


def _tn_plan(I, J, groups, rpg, Rr, mode):
    splits, cps = _lib.tc_gemm_tn_plan(I, J, groups, rpg, mode)
    chunk = 32 if mode < 2 else 64
    cpg = -(-rpg // chunk)
    bn = 64 if J <= 64 else 128
    return dict(splits=splits, cps=cps, cpg=cpg, total=groups * cpg, flush=128 // chunk, R=Rr,
                bn=bn, tiles=-(-I // 128) * -(-J // bn), sms=_lib.device_info()["sms"])


def _check_regime(regime, plan, mode):
    for tag in regime.split():
        name, _, modes = tag.partition(":")
        if not modes or str(mode) in modes:
            assert _REGIMES[name](plan), "regime %r not reached in mode %d: %s" % (name, mode, plan)


TN_CASES = [
    # I, J, groups, rpg, lda, pitchA, offA, R, pitchB, acc, ldc, regime
    _legacy(10, 64, 1280, 3, 100, 64, 103, 1, 640, 102, 0, 1280, "one"),
    _legacy(10, 128, 704, 2, 200, 128, 210, 5, 128, 206, 0, 704, "one"),
    _legacy(10, 2048, 288, 2, 131, 2048, 131, 0, 32, 140, 0, 288, "one"),      # folded sinc wgrad
    _legacy(10, 512, 5632, 4, 25, 512, 35, 5, 1024, 30, 0, 5632, "one"),
    _legacy(10, 256, 1920, 1, 300, 256, 300, 0, 1920, 300, 1, 1920, "one"),
    _legacy(10, 100, 512, 1, 77, 100, 77, 0, 512, 77, 0, 515, "one"),          # I tail, odd ldc
    (64, 1280, 3, 433, 64, 440, 3, 640, 437, 0, 1280, "2-8 mid uneven unfolded"),
    (128, 704, 1, 1025, 128, 1025, 0, 128, 1025, 1, 704, "2-8 mid uneven unfolded"),   # accumulate
    (128, 704, 5, 1617, 128, 1630, 7, 128, 1620, 0, 736, ">16 mid uneven"),   # ldc > J
    (128, 704, 4, 2838, 128, 2840, 1, 64, 2850, 1, 704, ">16 unfolded unblocked"),
    (128, 64, 5, 900, 128, 905, 2, 64, 903, 0, 96, "bn64 mid uneven"),
    (100, 512, 3, 700, 104, 700, 0, 512, 704, 0, 512, "split mid uneven"),    # I tail 100
    (192, 256, 3, 700, 200, 710, 4, 256, 705, 1, 264, "split mid uneven"),    # I tail 192
    (1024, 2176, 3, 650, 1024, 650, 0, 2176, 652, 0, 2176, "capped"),
    # PASE+ weight gradients at N = 4, T = 32000: block-1 conv, block-2 conv, dWcat, QRNN dWq
    (64, 1280, 4, 3200, 64, 3203, 1, 640, 3202, 0, 1280, "split mid uneven"),
    (128, 704, 4, 1600, 128, 1610, 5, 128, 1605, 0, 704, ">16:01 split:23 mid"),
    (256, 1920, 1, 800, 256, 800, 0, 1920, 800, 0, 1920, "split:01 one:23"),
    (1536, 1024, 4, 200, 1536, 200, 0, 512, 201, 0, 1024, "one"),
]


def _tn_case(I, J, groups, rpg, lda, pitchA, offA, Rr, pitchB, ldc, mode, seed, alpha_dev=None,
             scale=None, poison=True):
    """Operands (mode format, unused memory poisoned) and the argument list of one TN call."""
    A = R(groups * pitchA * lda + I + 128, seed=seed)
    b_rows = groups * pitchB + (J + Rr - 1) // Rr + 2
    B = R(b_rows * Rr, seed=seed + 1)
    C = R(I * ldc, seed=seed + 2)
    (Ah, Al), (Bh, Bl) = _operands(A, mode, scale=scale), _operands(B, mode)
    if poison:
        # A: rows no (group, u) uses, and columns [I, lda) of every row (the kernel reads them
        # only for output rows >= I); B: folded rows outside every group's rows [0, rpg + J/R)
        row = torch.arange(A.numel()) // lda
        u = row % pitchA - offA
        used = (row < groups * pitchA) & (u >= 0) & (u < rpg)
        _poison((Ah, Al), ~used | (torch.arange(A.numel()) % lda >= I))
        brow = torch.arange(B.numel()) // Rr
        last = rpg - 1 + (J - 1) // Rr
        bused = torch.zeros(B.numel(), dtype=torch.bool)
        for g in range(groups):
            bused |= (brow >= g * pitchB) & (brow <= g * pitchB + last)
        _poison((Bh, Bl), ~bused)
    return [Ah, Al, lda, pitchA, offA, Bh, Bl, Rr, pitchB, b_rows, C, ldc, I, J, groups, rpg,
            0.25, alpha_dev, 0, mode]


def _tn_check(cpu, dev, mode, I, J, ldc):
    out_c, out_d = cpu[10].view(I, ldc), dev[10].cpu().view(I, ldc)
    # guard columns [J, ldc) keep their initial values in both
    assert torch.equal(out_c[:, J:], out_d[:, J:]), "columns past J were written"
    out_c, out_d = out_c[:, :J], out_d[:, :J]
    scale = float(out_c.abs().max())
    assert scale > 0
    tol = (4e-6 if mode in (1, 3) else 4e-5) * scale
    err = float((out_c - out_d).abs().max())
    assert err <= tol, "C max err %.3e > %.3e (mode %d)" % (err, tol, mode)


@pytest.mark.parametrize("mode", [1, 0, 3, 2])
@pytest.mark.parametrize("I,J,groups,rpg,lda,pitchA,offA,Rr,pitchB,acc,ldc,regime", TN_CASES)
def test_tc_gemm_tn(I, J, groups, rpg, lda, pitchA, offA, Rr, pitchB, acc, ldc, regime, mode):
    """Every case, in all four modes where the shape is legal; modes 2 and 3 take alpha
    through alpha_dev (3xF16: the operand is pre-scaled by the power of two it undoes)."""
    if mode >= 2 and (Rr % 64 or J % 64 or lda % 8):
        pytest.skip("16-bit modes need 128-byte rows (64 elements)")
    plan = _tn_plan(I, J, groups, rpg, Rr, mode)
    print("TN %dx%d groups %d rpg %d mode %d: splits %d, chunks per split %d"
          % (I, J, groups, rpg, mode, plan["splits"], plan["cps"]))
    _check_regime(regime, plan, mode)
    s = 2.0 ** 4
    alpha_dev = torch.tensor([1.0 / s, s]) if mode >= 2 else None
    args = _tn_case(I, J, groups, rpg, lda, pitchA, offA, Rr, pitchB, ldc, mode, 21,
                    alpha_dev=alpha_dev, scale=s if mode == 3 else None)
    args[18] = acc
    cpu, dev = _run("pase_tc_gemm_tn", args)
    _tn_check(cpu, dev, mode, I, J, ldc)


@pytest.mark.parametrize("I,J,groups,rpg,lda,pitchA,offA,Rr,pitchB", [
    (4096, 320, 2, 131, 4096, 131, 0, 64, 140),      # folded sinc wgrad (fold 64)
    (1536, 1024, 3, 40, 1536, 40, 0, 512, 41),       # QRNN gate weight gradient
    (64, 128, 2, 300, 64, 302, 1, 64, 301),          # block-1 dgrad-side shape, J = BN
])
@pytest.mark.parametrize("mode", [2, 3])
def test_tc_gemm_tn_16bit_shapes(I, J, groups, rpg, lda, pitchA, offA, Rr, pitchB, mode):
    """16-bit-only shapes (64-element folded rows) + the device-side alpha of a scaled
    gradient operand."""
    A = R(groups * pitchA * lda + I + 128, seed=41) * (1e-7 if mode == 3 else 1.0)
    b_rows = groups * pitchB + (J + Rr - 1) // Rr + 2
    B = R(b_rows * Rr, seed=42)
    C = torch.zeros(I * J)
    s = 2.0 ** 36 if mode == 3 else 1.0
    alpha_dev = torch.tensor([1.0 / s, s]) if mode == 3 else None
    (Ah, Al), (Bh, Bl) = _operands(A, mode, scale=s), _operands(B, mode)
    args = [Ah, Al, lda, pitchA, offA, Bh, Bl, Rr, pitchB, b_rows, C, J, I, J, groups, rpg, 1.0,
            alpha_dev, 0, mode]
    cpu, dev = _run("pase_tc_gemm_tn", args)
    out_c, out_d = cpu[10], dev[10].cpu()
    scale = float(out_c.abs().max())
    assert scale > 0
    tol = (4e-6 if mode == 3 else 4e-5) * scale
    err = float((out_c - out_d).abs().max())
    assert err <= tol, "C max err %.3e > %.3e (mode %d)" % (err, tol, mode)


_SPLIT_A = (64, 1280, 3, 433, 64, 440, 3, 640, 437, 1280)      # I, J, groups, rpg, lda, pitchA,
_SPLIT_B = (128, 704, 5, 1617, 128, 1630, 7, 128, 1620, 736)   # offA, R, pitchB, ldc


@pytest.mark.parametrize("mode", [1, 3])
def test_tc_gemm_tn_back_to_back(mode):
    """Two split calls of different shapes on one stream, no synchronisation between them:
    the second reuses the shared partial-tile workspace only after the first has reduced."""
    for shp in (_SPLIT_A, _SPLIT_B):
        assert _tn_plan(*shp[:4], shp[7], mode)["splits"] > 1
    runs = [_tn_case(*shp, mode, 50 + 10 * k) for k, shp in enumerate((_SPLIT_A, _SPLIT_B))]
    devs = [[a.cuda() if isinstance(a, torch.Tensor) else a for a in args] for args in runs]
    for dev in devs:
        _lib.call("pase_tc_gemm_tn", *dev)
    torch.cuda.synchronize()
    for args, dev, shp in zip(runs, devs, (_SPLIT_A, _SPLIT_B)):
        cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
        emul.call("pase_tc_gemm_tn", *cpu)
        _tn_check(cpu, dev, mode, shp[0], shp[1], shp[9])


@pytest.mark.parametrize("mode", [1, 2])
def test_tc_gemm_tn_graph_replay(mode):
    """A split TN captured in a CUDA graph and replayed twice with new operands copied into
    its input buffers: both replays match the spec."""
    shp = _SPLIT_B
    assert _tn_plan(*shp[:4], shp[7], mode)["splits"] > 1
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in
           _tn_case(*shp, mode, 70)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _lib.call("pase_tc_gemm_tn", *dev)          # warm-up: allocates the workspace
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        _lib.call("pase_tc_gemm_tn", *dev)
    for seed in (80, 90):
        new = _tn_case(*shp, mode, seed)
        for i in (0, 1, 5, 6, 10):
            if new[i] is not None:
                dev[i].copy_(new[i])
        g.replay()
        torch.cuda.synchronize()
        cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in new]
        emul.call("pase_tc_gemm_tn", *cpu)
        _tn_check(cpu, dev, mode, shp[0], shp[1], shp[9])


# ---- run-to-run reproducibility: the same call twice on identical inputs, equal bits ----
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_tc_gemm_tn_split_is_reproducible(mode):
    shp = (64, 1280, 4, 3200, 64, 3203, 1, 640, 3202, 1280)      # 13 splits
    assert _tn_plan(*shp[:4], shp[7], mode)["splits"] > 1
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in _tn_case(*shp, mode, 100)]
    outs = []
    for _ in range(2):
        c = dev[10].clone()
        _lib.call("pase_tc_gemm_tn", *(dev[:10] + [c] + dev[11:]))
        outs.append(c)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("mode", [1, 3])
def test_tc_gemm_nt_stats_reproducible(mode):
    """NT with BatchNorm statistics (fp64 block partials) and pase_bn_finalize on them: the
    fp64 sums agree to 1e-14 and the fp32 statistics derived from them are equal."""
    M, N, K, Rr, rows_in, t_valid, rows_out = 9000, 512, 640, 128, 1000, 990, 990
    a_rows = M + (K + Rr - 1) // Rr + 2
    A = R(a_rows * Rr, seed=111)
    B = R(N * K, seed=112, scale=0.1)
    (Ah, Al), (Bh, Bl) = _operands(A, mode), _operands(B, mode, weights=True)
    dA = [t.cuda() if t is not None else None for t in (Ah, Al, Bh, Bl)]
    groups = (M + rows_in - 1) // rows_in
    res = []
    for _ in range(2):
        C = torch.zeros(groups * rows_out * N, device="cuda")
        cs, cq = (torch.zeros(N, dtype=torch.float64, device="cuda") for _ in range(2))
        _lib.call("pase_tc_gemm_nt", dA[0], dA[1], a_rows, Rr, dA[2], dA[3], K, C, N, M, N, K,
                  1.0, None, None, rows_in, t_valid, rows_out, 1, cs, cq, 0, mode, 0)
        outs = [torch.zeros(N, device="cuda") for _ in range(4)]
        rm, rv = torch.zeros(N, device="cuda"), torch.ones(N, device="cuda")
        _lib.call("pase_bn_finalize", cs, cq, N, 1, float(groups * t_valid),
                  torch.ones(N, device="cuda"), torch.zeros(N, device="cuda"), rm, rv, 0.1, 1e-5,
                  *outs)
        res.append((C, cs, cq, outs, rm, rv))
    torch.cuda.synchronize()
    (C1, s1, q1, o1, rm1, rv1), (C2, s2, q2, o2, rm2, rv2) = res
    assert torch.equal(C1, C2)
    for a, b in ((s1, s2), (q1, q2)):
        assert float((a - b).abs().max()) <= 1e-14 * float(a.abs().max())
    for a, b in zip(o1 + [rm1, rv1], o2 + [rm2, rv2]):
        assert torch.equal(a, b)


def test_tc_gemm_nt_ctxmse_reproducible():
    """Fused regression-head output layer: the fp16 residual pair is equal, the fp64 loss and
    bias-gradient accumulators agree to 1e-14."""
    Bn, F, T, r, K = 4, 40, 700, 3, 256
    M, N, Rr, ldr = Bn * T, F * r, 256, 128
    a_rows = M + 3
    A, W = R(a_rows * Rr, seed=121), R(N * K, seed=122, scale=0.1)
    (Ah, Al), (Bh, Bl) = _operands(A, 3), _operands(W, 3, weights=True)
    d = [t.cuda() for t in (Ah, Al, Bh, Bl)]
    bias, label = R(N, seed=123).cuda(), R(Bn * F * T, seed=124).cuda()
    scale = torch.tensor([1.0 / 64, 64.0]).cuda()
    res = []
    for _ in range(2):
        rh, rl = (torch.zeros(M * ldr, dtype=torch.float16, device="cuda") for _ in range(2))
        loss = torch.zeros(1, dtype=torch.float64, device="cuda")
        db = torch.zeros(N, dtype=torch.float64, device="cuda")
        _lib.call("pase_tc_gemm_nt_ctxmse", d[0], d[1], a_rows, Rr, d[2], d[3], K, rh, rl, ldr,
                  M, N, K, bias, label, Bn, F, T, r, scale, loss, db)
        res.append((rh, rl, loss, db))
    torch.cuda.synchronize()
    (h1, l1, L1, d1), (h2, l2, L2, d2) = res
    assert torch.equal(h1, h2) and torch.equal(l1, l2)
    assert abs(float(L1) - float(L2)) <= 1e-14 * abs(float(L1))
    assert float((d1 - d2).abs().max()) <= 1e-14 * float(d1.abs().max())
    assert torch.equal(L1.float(), L2.float()) and torch.equal(d1.float(), d2.float())
