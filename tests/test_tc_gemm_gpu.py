"""wgmma / TMA GEMM kernels against the exact spec (the product of the operands as the
tensor core reads them, accumulated in fp64).  Modes 1 (3xTF32) and 3 (3xF16) must be
fp32-equivalent; mode 0 (TF32) and mode 2 (bf16) are exact products of rounded operands, so
they too are checked tightly against the spec evaluated on the SAME rounded operands."""
import pytest
import torch

import emul_ops
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
        emul_ops.pase_split_tf32(x, hi, lo, x.numel())
        return hi, lo
    emul_ops.pase_split_tf32(x, None, lo, x.numel())
    return x.clone(), lo


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
    xt = emul_ops._tf32_trunc(x)
    assert float((x - xt - lo_a).abs().max()) <= float(x.abs().max()) * 2.0 ** -21


NT_CASES = [
    # M, N, K, R, rows_in, t_valid, rows_out, fold, bias, stats, acc
    (256, 128, 128, 128, 256, 256, 256, 1, True, True, 0),        # one full tile, plain
    (1000, 64, 1280, 640, 103, 100, 100, 1, True, True, 0),       # block-1 like, k spans 2 rows
    (700, 128, 704, 128, 70, 64, 64, 1, True, True, 0),           # stride-2 k=11 shape
    (300, 256, 1408, 128, 300, 300, 300, 1, False, False, 0),     # BN=256
    (520, 2048, 288, 32, 130, 4100, 129, 32, False, True, 0),     # folded sinc (fold 32)
    (333, 512, 5632, 1024, 111, 100, 100, 1, True, False, 1),     # long K, accumulate
    (260, 1920, 256, 256, 260, 260, 260, 1, False, False, 0),     # dcat shape, wide N
    (300, 128, 200, 64, 300, 300, 300, 1, True, True, 0),         # K % 32 != 0: per-k-block kernel
    (4000, 256, 2816, 256, 1000, 990, 990, 1, True, True, 0),     # many tiles / persistent loop
]


@pytest.mark.parametrize("mode", [1, 0, 3, 2])
@pytest.mark.parametrize("M,N,K,Rr,rows_in,t_valid,rows_out,fold,bias,stats,acc", NT_CASES)
def test_tc_gemm_nt(M, N, K, Rr, rows_in, t_valid, rows_out, fold, bias, stats, acc, mode):
    if mode >= 2:
        if Rr % 64 or (K * 2) % 16:
            pytest.skip("16-bit modes need folded rows of 64 elements")
    a_rows = M + (K + Rr - 1) // Rr + 2
    A = R(a_rows * Rr, seed=11)
    B = R(N * K, seed=12, scale=0.1)
    groups = (M + rows_in - 1) // rows_in
    C = R(groups * rows_out * N + 8, seed=13)
    bs = R(N, seed=14) if bias else None
    cs = torch.zeros(N, dtype=torch.float64) if stats else None
    cq = torch.zeros(N, dtype=torch.float64) if stats else None
    (Ah, Al), (Bh, Bl) = _operands(A, mode), _operands(B, mode, weights=True)
    args = [Ah, Al, a_rows, Rr, Bh, Bl, K, C, N, M, N, K, 0.5, None, bs, rows_in, t_valid,
            rows_out, fold, cs, cq, acc, mode, 0]
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul_ops.call("pase_tc_gemm_nt", *cpu)
    _lib.call("pase_tc_gemm_nt", *dev)
    torch.cuda.synchronize()
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
@pytest.mark.parametrize("M,N,K,Rr,rows_in,t_valid,rows_out,fold", [
    (1000, 64, 1280, 640, 103, 100, 100, 1),        # BN=64, 1-CTA
    (700, 128, 704, 128, 70, 64, 64, 1),            # BN=128
    (520, 4096, 320, 64, 130, 8200, 129, 64),       # folded sinc (fold 64), wide N, stats
    (300, 256, 5632, 1024, 300, 300, 300, 1),       # 256-wide tiles (mode 2) / pair (mode 3)
])
def test_tc_gemm_nt_bf16_out_and_alpha_dev(M, N, K, Rr, rows_in, t_valid, rows_out, fold, mode):
    """bf16 output (C rounded once from the fp32 result) and the device-side alpha that
    undoes a power-of-two operand scale (3xF16 gradients)."""
    a_rows = M + (K + Rr - 1) // Rr + 2
    A = R(a_rows * Rr, seed=31) * (1e-6 if mode == 3 else 1.0)     # tiny gradients
    B = R(N * K, seed=32, scale=0.1)
    groups = (M + rows_in - 1) // rows_in
    s = 2.0 ** 32 if mode == 3 else 1.0
    alpha_dev = torch.tensor([1.0 / s, s]) if mode == 3 else None
    (Ah, Al), (Bh, Bl) = _operands(A, mode, scale=s), _operands(B, mode, weights=True)
    cs, cq = torch.zeros(N, dtype=torch.float64), torch.zeros(N, dtype=torch.float64)
    for c16 in ((1, 0) if mode != 1 else (1,)):
        C = torch.zeros(groups * rows_out * N + 8, dtype=torch.bfloat16 if c16 else torch.float32)
        args = [Ah, Al, a_rows, Rr, Bh, Bl, K, C, N, M, N, K, 1.0, alpha_dev, None, rows_in,
                t_valid, rows_out, fold, cs.clone(), cq.clone(), 0, mode, c16]
        cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
        dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
        emul_ops.call("pase_tc_gemm_nt", *cpu)
        _lib.call("pase_tc_gemm_nt", *dev)
        torch.cuda.synchronize()
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


TN_CASES = [
    # I, J, groups, rpg, lda, pitchA, offA, R, pitchB, acc
    (64, 1280, 3, 100, 64, 103, 1, 640, 102, 0),
    (128, 704, 2, 200, 128, 210, 5, 128, 206, 0),
    (2048, 288, 2, 131, 2048, 131, 0, 32, 140, 0),        # folded sinc wgrad
    (512, 5632, 4, 25, 512, 35, 5, 1024, 30, 0),
    (256, 1920, 1, 300, 256, 300, 0, 1920, 300, 1),
    (100, 512, 1, 77, 100, 77, 0, 512, 77, 0),            # I tail (emb 100)
]


@pytest.mark.parametrize("mode", [1, 0, 3, 2])
@pytest.mark.parametrize("I,J,groups,rpg,lda,pitchA,offA,Rr,pitchB,acc", TN_CASES)
def test_tc_gemm_tn(I, J, groups, rpg, lda, pitchA, offA, Rr, pitchB, acc, mode):
    if mode >= 2 and (Rr % 64 or J % 64 or lda % 8):
        pytest.skip("16-bit modes need 128-byte rows (64 elements)")
    A = R(groups * pitchA * lda + I + 128, seed=21)
    b_rows = groups * pitchB + (J + Rr - 1) // Rr + 2
    B = R(b_rows * Rr, seed=22)
    C = R(I * J, seed=23)
    (Ah, Al), (Bh, Bl) = _operands(A, mode), _operands(B, mode)
    args = [Ah, Al, lda, pitchA, offA, Bh, Bl, Rr, pitchB, b_rows, C, J, I, J, groups, rpg, 0.25,
            None, acc, mode]
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul_ops.call("pase_tc_gemm_tn", *cpu)
    _lib.call("pase_tc_gemm_tn", *dev)
    torch.cuda.synchronize()
    out_c, out_d = cpu[10], dev[10].cpu()
    scale = float(out_c.abs().max())
    tol = (4e-6 if mode in (1, 3) else 4e-5) * max(scale, 1.0)
    err = float((out_c - out_d).abs().max())
    assert err <= tol, "C max err %.3e > %.3e (mode %d)" % (err, tol, mode)


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
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul_ops.call("pase_tc_gemm_tn", *cpu)
    _lib.call("pase_tc_gemm_tn", *dev)
    torch.cuda.synchronize()
    out_c, out_d = cpu[10], dev[10].cpu()
    scale = float(out_c.abs().max())
    assert scale > 0
    tol = (4e-6 if mode == 3 else 4e-5) * scale
    err = float((out_c - out_d).abs().max())
    assert err <= tol, "C max err %.3e > %.3e (mode %d)" % (err, tol, mode)
