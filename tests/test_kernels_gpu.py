"""Every C-ABI kernel, called through ctypes on the GPU, against its torch
semantic spec (tests/emul/) on identical random inputs."""
import pytest
import torch

import emul
from pase_b200 import _lib

pytestmark = pytest.mark.gpu


def run_both(name, args, rtol=1e-4, atol=1e-5, cmp_scale=None, skip=()):
    """args: list of tensors (CPU) / scalars / None.  Runs the emulation on clones and the
    CUDA kernel on device copies; compares every tensor argument afterwards."""
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul.call(name, *cpu)
    _lib.call(name, *dev)
    torch.cuda.synchronize()
    for i, (c, d) in enumerate(zip(cpu, dev)):
        if not isinstance(c, torch.Tensor) or i in skip:
            continue
        d = d.cpu()
        if c.dtype in (torch.float64, torch.bfloat16, torch.float16):
            c, d = c.float(), d.float()
        scale = max(float(c.abs().max()), 1.0) if cmp_scale is None else cmp_scale
        err = (c - d).abs()
        tol = atol * scale + rtol * c.abs()
        assert bool((err <= tol).all()), "%s arg %d: max err %.3e (scale %.3e)" % (
            name, i, float(err.max()), scale)
    return cpu, dev


def R(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return scale * torch.randn(*shape, generator=g)


@pytest.mark.parametrize("M,N,K,lda,rows_in,t_valid,rows_out,fold,bias,stats,acc", [
    (300, 64, 256, 256, 300, 300, 300, 1, True, True, 0),          # plain, BN=64 tile
    (517, 128, 704, 128, 47, 40, 40, 1, True, True, 0),            # overlapping view, row groups
    (260, 256, 256, 4, 65, 250, 63, 4, False, True, 0),            # folded sinc shape
    (129, 100, 512, 512, 129, 129, 129, 1, True, False, 0),        # N tail (emb 100)
    (200, 85, 256, 256, 200, 200, 200, 1, True, False, 1),         # accumulate, odd N + ldc
    (1030, 640, 128, 64, 103, 101, 101, 1, False, False, 0),       # dgrad shape
])
def test_gemm_nt(M, N, K, lda, rows_in, t_valid, rows_out, fold, bias, stats, acc):
    A = R(M * lda + K + 8, seed=1)
    B = R(N * K, seed=2, scale=0.1)
    groups = (M + rows_in - 1) // rows_in
    ldc = N if N % 4 == 0 else N + 1
    C = R(groups * rows_out * ldc + 8, seed=3)
    bs = R(N, seed=4) if bias else None
    cs = torch.zeros(N, dtype=torch.float64) if stats else None
    cq = torch.zeros(N, dtype=torch.float64) if stats else None
    run_both("pase_gemm_nt", [A, lda, B, K, C, ldc, M, N, K, 0.5, bs, rows_in, t_valid, rows_out,
                              fold, cs, cq, acc], rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("I,J,groups,rpg,lda,pitchA,offA,ldb,pitchB,offB,acc", [
    (64, 1280, 3, 100, 64, 103, 1, 640, 102, 0, 0),
    (256, 256, 2, 500, 256, 500, 0, 4, 520, 0, 0),
    (100, 1920, 1, 77, 100, 77, 0, 1920, 77, 0, 1),
    (512, 64, 4, 33, 512, 40, 5, 64, 33, 0, 0),
    (128, 704, 4, 1600, 128, 1610, 5, 704, 1605, 3, 1),     # ~66 splits, accumulate
    (100, 60, 3, 900, 100, 905, 2, 60, 903, 1, 0),          # BN=64 tile, tails, splits
    # 16 x 17 = 272 tiles: ceil(3 SMs / tiles) = 2 splits would overflow the 4 x SMs-tile
    # workspace on a 132-SM H100; the launcher keeps splits x tiles within it
    (2048, 2176, 2, 128, 2048, 130, 1, 2176, 129, 0, 0),
])
def test_gemm_tn(I, J, groups, rpg, lda, pitchA, offA, ldb, pitchB, offB, acc):
    A = R(groups * pitchA * lda + I + 8, seed=5)
    B = R(groups * pitchB * ldb + J + 8, seed=6)
    C = R(I * J, seed=7)
    run_both("pase_gemm_tn", [A, lda, pitchA, offA, B, ldb, pitchB, offB, C, J, I, J, groups, rpg,
                              0.25, acc], rtol=2e-4, atol=2e-5)


# ---- run-to-run reproducibility: the same computation twice on identical inputs ----
def _twice(name, args, outs):
    """Run `name` twice on fresh device copies of args; -> the two lists of outputs."""
    res = []
    for _ in range(2):
        dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
        _lib.call(name, *dev)
        res.append([dev[i] for i in outs])
    torch.cuda.synchronize()
    return res


def _same_fp64(a, b):
    """fp64 accumulators: equal to 1e-14, and equal once rounded to fp32 (what consumers use)."""
    assert float((a - b).abs().max()) <= 1e-14 * float(a.abs().max())
    assert torch.equal(a.float(), b.float())


def test_gemm_tn_is_reproducible():
    I, J, groups, rpg, lda, pitchA, offA, ldb, pitchB = 128, 704, 4, 1600, 128, 1610, 5, 704, 1605
    A = R(groups * pitchA * lda + I + 8, seed=61)
    B = R(groups * pitchB * ldb + J + 8, seed=62)
    (c1,), (c2,) = _twice("pase_gemm_tn", [A, lda, pitchA, offA, B, ldb, pitchB, 0,
                                           torch.zeros(I * J), J, I, J, groups, rpg, 1.0, 0], [8])
    assert torch.equal(c1, c2)


def test_bn_prelu_bwd_and_colsum_are_reproducible():
    N, T, C, padL, padR, pool_d = 4, 1603, 128, 5, 5, 8
    Tp = T + padL + padR
    y = R(N * T * C, seed=63)
    mean, invstd = R(C, seed=64, scale=0.1), R(C, seed=65).abs() + 0.5
    scale, shift, alpha = R(C, seed=66), R(C, seed=67), R(C, seed=68, scale=0.3)
    pool_T = T // pool_d
    args = [y, 0, T * C, N, T, C, mean, invstd, scale, shift, alpha, R(N * Tp * C, seed=69), 0,
            Tp * C, C, padL, padR, None, 0, 0, 0, R(N * pool_T * C, seed=70), pool_T * C, C,
            pool_d, pool_T, torch.zeros(N * T * C), T * C] + \
        [torch.zeros(C, dtype=torch.float64) for _ in range(3)] + [torch.zeros(2)]
    r1, r2 = _twice("pase_bn_prelu_bwd_reduce", args, [26, 28, 29, 30, 31])
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[4], r2[4])
    for a, b in zip(r1[1:4], r2[1:4]):
        _same_fp64(a, b)
    outs = []
    for du, s1, s2 in ((r1[0], r1[1], r1[2]), (r2[0], r2[1], r2[2])):
        dy = torch.zeros_like(du)
        db = torch.zeros(C, dtype=torch.float64, device="cuda")
        _lib.call("pase_bn_prelu_bwd_apply", y.cuda(), 0, T * C, N, T, C, mean.cuda(),
                  invstd.cuda(), R(C, seed=71).cuda(), s1, s2, float(N * T), du, dy, None, 0,
                  T * C, db, None, None)
        outs.append((dy, db))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0])
    _same_fp64(outs[0][1], outs[1][1])
    rows = 20000
    (s1,), (s2,) = _twice("pase_colsum", [R(rows * 520, seed=72), 520, rows, 517,
                                          torch.zeros(517, dtype=torch.float64)], [4])
    _same_fp64(s1, s2)


# ---- small helpers of the 3xF16 gradient scaling and of the flat-gradient packing ----
def test_bound_scale_bit_exact():
    """{1/s, s} with s the power of two placing 1.0001 x (a0 a1 + a2 + a3) below 2^14,
    including bounds that are exact powers of two, zero and tiny / huge bounds."""
    for a4 in ([2.0, 4.0, 0.0, 0.0], [0.5, 0.5, 0.0, 0.0], [1.0, 2.0 ** -20, 0.0, 0.0],
               [2.0 ** 14, 1.0, 0.0, 0.0], [1.0, 1.0, 2.0 ** 15, 2.0 ** 15], [3.0, 5.0, 1.0, 0.5],
               [0.0, 0.0, 0.0, 0.0], [1e-20, 1e-10, 0.0, 0.0], [1e19, 1e19, 0.0, 0.0],
               [0.1, 0.3, 7.0, 1e-3]):
        cpu, dev = run_both("pase_bound_scale", [torch.tensor(a4), torch.zeros(2)], rtol=0, atol=0)
        assert torch.equal(cpu[1], dev[1].cpu()), (a4, cpu[1], dev[1])


@pytest.mark.parametrize("rows,cols,ld", [(1, 1, 1), (300, 37, 40), (1000, 1001, 1003),
                                          (64, 4, 4), (5000, 99, 128)])
def test_rownorm_max(rows, cols, ld):
    """max_r ||X[r, :cols]|| over rows spanning 20 decades, with in-row spikes; cols not a
    multiple of 4 and ld > cols (the padding holds large values that must be ignored)."""
    g = torch.Generator().manual_seed(rows + cols)
    X = torch.randn(rows, ld, generator=g)
    X *= 10.0 ** torch.randint(-10, 10, (rows, 1), generator=g).float()
    X[::7, 0] *= 1e4
    X[:, cols:] = 1e30
    for prior in (0.0, float(X[:, :cols].double().norm(dim=1).max()) * 2):
        amax = torch.tensor([prior])
        cpu, dev = run_both("pase_rownorm_max", [X.reshape(-1), ld, rows, cols, amax],
                            rtol=1e-5, atol=0)
        if prior:
            assert float(dev[4][0]) == float(amax[0])


@pytest.mark.parametrize("njobs", [7, 128])
def test_scatter_copy(njobs):
    """Strided 2-D copies of several shapes in one launch (128 = the table's capacity); the
    guard elements between destinations stay untouched."""
    g = torch.Generator().manual_seed(njobs)
    shapes = [(1, 1, 1, 1), (3, 5, 7, 6), (17, 33, 40, 35), (64, 100, 100, 100),
              (2, 1000, 1003, 1001), (1, 4097, 4097, 4097), (9, 2, 2, 9)]
    while len(shapes) < njobs:
        r, c = (int(v) for v in torch.randint(1, 40, (2,), generator=g))
        shapes.append((r, c, c + int(torch.randint(0, 4, (1,), generator=g)),
                       c + int(torch.randint(0, 4, (1,), generator=g))))
    so, do, s_off, d_off = 0, 0, [], []
    for (r, c, sl, dl) in shapes:
        s_off.append(so)
        d_off.append(do + 3)                       # 3 guard elements before every destination
        so += (r - 1) * sl + c + 5
        do += 3 + (r - 1) * dl + c + 3
    src = torch.randn(so, generator=g)
    dst = torch.full((do,), -7.0)
    ref = dst.clone()
    srcd, dstd = src.cuda(), dst.cuda()
    total = sum(r * c for (r, c, _, _) in shapes)

    def table(s, d):
        return torch.tensor([[s.data_ptr() + 4 * so_, d.data_ptr() + 4 * do_, r, c, sl, dl]
                             for (r, c, sl, dl), so_, do_ in zip(shapes, s_off, d_off)],
                            dtype=torch.int64).reshape(-1)
    emul.core.pase_scatter_copy(table(src, ref), njobs, total)
    _lib.call("pase_scatter_copy", table(srcd, dstd).cuda(), njobs, total)
    torch.cuda.synchronize()
    out = dstd.cpu()
    assert torch.equal(out, ref)
    assert int((out == -7.0).sum()) == do - total


def test_weight_layouts():
    Cout, Cin, k, s = 24, 16, 11, 2
    taps = -(-k // s)
    W = R(Cout * Cin * k, seed=8)
    run_both("pase_conv_w_to_fwd", [W, torch.zeros(Cout * Cin * k), Cout, Cin, k])
    run_both("pase_conv_w_from_fwd", [W, torch.zeros(Cout * Cin * k), Cout, Cin, k])
    run_both("pase_conv_w_to_dgrad", [W, torch.zeros(s * Cin * taps * Cout), Cout, Cin, k, s, taps])
    k2, s2 = 30, 4
    t2 = -(-k2 // s2)
    Wd = R(Cin * Cout * k2, seed=9)
    run_both("pase_deconv_w_to_fwd", [Wd, torch.zeros(s2 * Cout * t2 * Cin), Cin, Cout, k2, s2, t2])
    run_both("pase_deconv_w_from_fwd", [R(s2 * Cout * t2 * Cin, seed=10),
                                        torch.zeros(Cin * Cout * k2), Cin, Cout, k2, s2, t2])
    run_both("pase_deconv_w_to_bwd", [Wd, torch.zeros(Cin * Cout * k2), Cin, Cout, k2])
    run_both("pase_transpose_pad", [R(37 * 21, seed=11), 21, torch.zeros(21 * 40), 40, 37, 21])


def test_sinc_make_and_grad():
    from pase_b200.encoder import sinc_constants
    from detweights import fill_state_dict
    C, k, fold, Kv = 64, 251, 4, 256
    sd = fill_state_dict({"blocks.0.conv.low_hz_": torch.zeros(C, 1),
                          "blocks.0.conv.band_hz_": torch.zeros(C, 1)}, 3)
    low, band = sd["blocks.0.conv.low_hz_"].reshape(-1), sd["blocks.0.conv.band_hz_"].reshape(-1)
    band[5] = 9000.0          # forces the clamp at sr/2
    low[7] = -low[7]          # abs() branch
    n_, win = sinc_constants(k, 16000, "cpu")
    run_both("pase_sinc_make", [low, band, n_, win, torch.zeros(C * k), torch.zeros(fold * C * Kv),
                                C, k, fold, Kv, 50.0, 50.0, 16000.0], rtol=2e-3, atol=2e-5)
    dWp = R(fold * C * Kv, seed=12)
    run_both("pase_sinc_grad", [dWp, low, band, n_, win, torch.zeros(C), torch.zeros(C), C, k, fold,
                                Kv, 50.0, 50.0, 16000.0], rtol=5e-3, atol=2e-4)


def test_reflect_pad_and_bn_finalize():
    N, T = 3, 700
    run_both("pase_reflect_pad_wave", [R(N * T, seed=13), torch.zeros(N * 960), None, 0, N, T, 125,
                                       125, 960])
    # operand formats: tf32 residual twin, bf16, fp16 pair (bit-exact element-wise maps)
    x = R(N * T, seed=13) * 3.0
    for fmt, dt in ((0, torch.float32), (1, torch.bfloat16), (2, torch.float16)):
        dst = torch.zeros(N * 960, dtype=dt)
        lo = torch.zeros(N * 960, dtype=dt) if fmt != 1 else None
        cpu, dev = run_both("pase_reflect_pad_wave", [x, dst, lo, fmt, N, T, 125, 125, 960],
                            rtol=0, atol=0)
        assert torch.equal(cpu[1], dev[1].cpu())
        if lo is not None:
            assert torch.equal(cpu[2], dev[2].cpu())
    C, fold = 48, 4
    cs = R(C * fold, seed=14).double() * 100
    cq = (R(C * fold, seed=15).double().abs() + 1.0) * 5000
    run_both("pase_bn_finalize", [cs, cq, C, fold, 4000.0, R(C, seed=16), R(C, seed=17),
                                  R(C, seed=18), R(C, seed=19).abs(), 0.1, 1e-5, torch.zeros(C),
                                  torch.zeros(C), torch.zeros(C), torch.zeros(C)])
    run_both("pase_bn_eval_affine", [R(C, seed=18), R(C, seed=19).abs() + 0.1, R(C, seed=16), None,
                                     C, 1e-5, torch.zeros(C), torch.zeros(C), torch.zeros(C),
                                     torch.zeros(C)])


@pytest.mark.parametrize("with_lo", [False, True])
@pytest.mark.parametrize("N,T,C,padL,padR,pool_d", [(2, 203, 64, 4, 5, 16), (3, 77, 48, 0, 0, 0),
                                                    (2, 1001, 128, 5, 5, 8), (2, 50, 512, 9, 10, 2)])
def test_bn_prelu_pad_fwd(N, T, C, padL, padR, pool_d, with_lo):
    Tp = T + padL + padR
    y = R(N * (T + 3) * C, seed=20)
    d_rs = C + 8
    dst = torch.zeros(N * (Tp + 2) * d_rs)
    pool_T = T // pool_d if pool_d else 0
    pool = torch.zeros(N * max(pool_T, 1) * 200 + C) if pool_d else None
    cpu, dev = run_both("pase_bn_prelu_pad_fwd", [
        y, 0, (T + 3) * C, N, T, C, R(C, seed=21), R(C, seed=22), R(C, seed=23, scale=0.3), dst,
        torch.zeros_like(dst) if with_lo else None, 0,
        (Tp + 2) * d_rs, d_rs, padL, padR, pool, max(pool_T, 1) * 200, 200, pool_d, pool_T],
        skip=(10,))
    if with_lo:
        # the residual is a discontinuous function of the last bits of dst, so it is checked
        # against the GPU's own dst: trunc_tf32(dst) + lo == dst to 2^-21
        d, lo = dev[9].cpu(), dev[10].cpu()
        rec = emul.core._tf32_trunc(d) + lo
        assert float((rec - d).abs().max()) <= float(d.abs().max()) * 2.0 ** -21
        assert torch.equal(lo, emul.core._residual(d))


@pytest.mark.parametrize("y_bf16,fmt", [(1, 1), (0, 2), (1, 0), (0, 1)])
@pytest.mark.parametrize("N,T,C,padL,padR,pool_d", [(2, 203, 64, 4, 5, 16), (2, 1001, 128, 5, 5, 8),
                                                    (2, 50, 512, 9, 10, 2)])
def test_bn_prelu_pad_fwd_16bit(N, T, C, padL, padR, pool_d, y_bf16, fmt):
    """bf16 y and/or bf16 / fp16-pair operand output.  The stored value is a discontinuous
    function of the fp32 result near rounding boundaries: the bf16 output is compared at one
    bf16 ulp, the fp16 pair through the value it encodes (hi + lo/2^11) at fp32 accuracy."""
    Tp = T + padL + padR
    y = R(N * (T + 3) * C, seed=20)
    if y_bf16:
        y = y.to(torch.bfloat16)
    d_rs = C + 8
    dt = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}[fmt]
    dst = torch.zeros(N * (Tp + 2) * d_rs, dtype=dt)
    lo = torch.zeros_like(dst) if fmt == 2 else None
    pool_T = T // pool_d
    pool = torch.zeros(N * pool_T * 200 + C)
    args = [y, y_bf16, (T + 3) * C, N, T, C, R(C, seed=21), R(C, seed=22),
            R(C, seed=23, scale=0.3), dst, lo, fmt, (Tp + 2) * d_rs, d_rs, padL, padR, pool,
            pool_T * 200, 200, pool_d, pool_T]
    cpu = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul.call("pase_bn_prelu_pad_fwd", *cpu)
    _lib.call("pase_bn_prelu_pad_fwd", *dev)
    torch.cuda.synchronize()
    if fmt == 2:
        vc = cpu[9].float() + cpu[10].float() / 2048.0
        vd = dev[9].cpu().float() + dev[10].cpu().float() / 2048.0
        tol = 2e-6
    else:
        vc, vd = cpu[9].float(), dev[9].cpu().float()
        tol = 2.0 ** -7 if fmt == 1 else 2e-6
    err = (vc - vd).abs()
    assert bool((err <= tol * vc.abs() + 1e-6).all()), float(err.max())
    # pooled values: one differently-rounded bf16 element moves a window mean by ulp/pool_d
    assert float((cpu[16] - dev[16].cpu()).abs().max()) <= (2e-2 if fmt == 1 else 2e-5)


@pytest.mark.parametrize("N,T,C,padL,padR,pool_d,useB", [(2, 203, 64, 4, 5, 16, False),
                                                         (3, 77, 48, 0, 0, 0, True),
                                                         (2, 40, 512, 9, 10, 2, False)])
def test_bn_prelu_bwd(N, T, C, padL, padR, pool_d, useB):
    Tp = T + padL + padR
    y = R(N * T * C, seed=24)
    mean, invstd = R(C, seed=25, scale=0.1), R(C, seed=26).abs() + 0.5
    scale, shift, alpha = R(C, seed=27), R(C, seed=28), R(C, seed=29, scale=0.3)
    srcA = R(N * Tp * C, seed=30)
    srcB = R(N * T * 2 * C, seed=31) if useB else None
    pool_T = T // pool_d if pool_d else 0
    pool = R(N * max(pool_T, 1) * C, seed=32) if pool_d else None
    dst = torch.zeros(N * T * C)
    S1, S2, dal = (torch.zeros(C, dtype=torch.float64) for _ in range(3))
    amax = torch.zeros(2)
    cpu, dev = run_both("pase_bn_prelu_bwd_reduce", [
        y, 0, T * C, N, T, C, mean, invstd, scale, shift, alpha, srcA, 0, Tp * C, C, padL, padR,
        srcB, T * 2 * C, 2 * C, 1, pool, max(pool_T, 1) * C, C, pool_d, pool_T, dst, T * C,
        S1, S2, dal, amax], rtol=2e-4, atol=2e-5)
    du, s1, s2, am = cpu[26], cpu[28], cpu[29], cpu[31]
    assert float(am[0]) > 0 and float(am[1]) > 0
    gamma = R(C, seed=33)
    run_both("pase_bn_prelu_bwd_apply", [y, 0, T * C, N, T, C, mean, invstd, gamma, s1, s2,
                                         float(N * T), du, du.clone(), None, 0, T * C,
                                         torch.zeros(C, dtype=torch.float64), None, None],
             rtol=2e-4, atol=2e-5)
    # fp16-pair output: dy scaled by the power of two derived from the bound; the pair must
    # encode s*dy at fp32 accuracy and stay far inside fp16's range
    hi, lo = torch.zeros(N * T * C, dtype=torch.float16), torch.zeros(N * T * C, dtype=torch.float16)
    sc = torch.zeros(2)
    args = [y, 0, T * C, N, T, C, mean, invstd, gamma, s1, s2, float(N * T), du, hi, lo, 2, T * C,
            torch.zeros(C, dtype=torch.float64), am, sc]
    cpu2 = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev2 = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul.call("pase_bn_prelu_bwd_apply", *cpu2)
    _lib.call("pase_bn_prelu_bwd_apply", *dev2)
    torch.cuda.synchronize()
    assert torch.equal(cpu2[19], dev2[19].cpu()), (cpu2[19], dev2[19])
    s = float(cpu2[19][1])
    vc = cpu2[13].float() + cpu2[14].float() / 2048.0
    vd = dev2[13].cpu().float() + dev2[14].cpu().float() / 2048.0
    assert float(vd.abs().max()) <= 16384.0 and float(vd.abs().max()) >= 16384.0 / 64
    assert float((vc - vd).abs().max()) <= 2e-5 * float(vc.abs().max())
    ref = torch.zeros(N * T * C)
    emul.call("pase_bn_prelu_bwd_apply", y, 0, T * C, N, T, C, mean, invstd, gamma, s1, s2,
              float(N * T), du, ref, None, 0, T * C, None, None, None)
    assert float((vd / s - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


@pytest.mark.parametrize("N,T,C,padL,padR,pool_d,useB,fmt", [
    (2, 203, 64, 4, 5, 16, False, 0), (3, 77, 48, 0, 0, 0, True, 0), (2, 40, 512, 9, 10, 2, False, 2),
    (2, 1603, 128, 5, 5, 8, False, 2), (3, 331, 256, 4, 5, 0, True, 2), (2, 203, 64, 4, 5, 16, False, 1),
    (2, 77, 64, 0, 0, 0, True, 1)])
def test_bn_prelu_bwd_no_du(N, T, C, padL, padR, pool_d, useB, fmt):
    """Sums-only pass 1 (dst = NULL) + pass 2 that recomputes du from the gradient sources
    (pase_bn_prelu_bwd_apply_src) against the spec, in the fp32 / fp16-pair / bf16 formats."""
    bf = fmt == 1
    Tp = T + padL + padR
    ydt = torch.bfloat16 if bf else torch.float32
    y = R(N * T * C, seed=24).to(ydt)
    mean, invstd = R(C, seed=25, scale=0.1), R(C, seed=26).abs() + 0.5
    scale, shift, alpha = R(C, seed=27), R(C, seed=28), R(C, seed=29, scale=0.3)
    a_bf = bf and not useB                 # the last block's source is fp32 in every mode
    srcA = R(N * Tp * C, seed=30).to(torch.bfloat16 if a_bf else torch.float32)
    srcB = R(N * T * 2 * C, seed=31) if useB else None
    pool_T = T // pool_d if pool_d else 0
    pool = R(N * max(pool_T, 1) * C, seed=32) if pool_d else None
    S1, S2, dal = (torch.zeros(C, dtype=torch.float64) for _ in range(3))
    amax = torch.zeros(2)
    src = [srcA, int(a_bf), Tp * C, C, padL, padR, srcB, T * 2 * C, 2 * C, 1, pool,
           max(pool_T, 1) * C, C, pool_d, pool_T]
    cpu, dev = run_both("pase_bn_prelu_bwd_reduce", [
        y, int(bf), T * C, N, T, C, mean, invstd, scale, shift, alpha] + src +
        [None, T * C, S1, S2, dal, amax], rtol=2e-4, atol=2e-5)
    s1, s2, am = cpu[28], cpu[29], cpu[31]
    gamma = R(C, seed=33)
    odt = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}[fmt]
    hi = torch.zeros(N * T * C, dtype=odt)
    lo = torch.zeros(N * T * C, dtype=odt) if fmt == 2 else None
    sc = torch.zeros(2)
    args = [y, int(bf), T * C, N, T, C, mean, invstd, gamma, scale, shift, alpha, s1, s2,
            float(N * T)] + src + [hi, lo, fmt, T * C, torch.zeros(C, dtype=torch.float64),
                                   am if fmt == 2 else None, sc if fmt == 2 else None]
    cpu2 = [a.clone() if isinstance(a, torch.Tensor) else a for a in args]
    dev2 = [a.cuda() if isinstance(a, torch.Tensor) else a for a in args]
    emul.call("pase_bn_prelu_bwd_apply_src", *cpu2)
    _lib.call("pase_bn_prelu_bwd_apply_src", *dev2)
    torch.cuda.synchronize()
    i_hi, i_lo, i_db, i_sc = 30, 31, 34, 36
    if fmt == 2:
        assert torch.equal(cpu2[i_sc], dev2[i_sc].cpu())
        vc = cpu2[i_hi].float() + cpu2[i_lo].float() / 2048.0
        vd = dev2[i_hi].cpu().float() + dev2[i_lo].cpu().float() / 2048.0
        assert float(vd.abs().max()) <= 16384.0
        tol = 2e-5
    else:
        vc, vd = cpu2[i_hi].float(), dev2[i_hi].cpu().float()
        tol = 2.0 ** -7 if bf else 2e-5
    assert float((vc - vd).abs().max()) <= tol * float(vc.abs().max())
    db_c, db_d = cpu2[i_db], dev2[i_db].cpu()
    assert float((db_c - db_d).abs().max()) <= 1e-4 * float(db_c.abs().max()) + 1e-6
    if not bf:
        # identical to the two-pass form with a stored du
        du = torch.zeros(N * T * C)
        emul.call("pase_bn_prelu_bwd_reduce", y, 0, T * C, N, T, C, mean, invstd, scale, shift,
                  alpha, *src, du, T * C, torch.zeros(C, dtype=torch.float64),
                  torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64), None)
        ref = torch.zeros(N * T * C)
        emul.call("pase_bn_prelu_bwd_apply", y, 0, T * C, N, T, C, mean, invstd, gamma, s1, s2,
                  float(N * T), du, ref, None, 0, T * C, None, None, None)
        s = float(cpu2[i_sc][1]) if fmt == 2 else 1.0
        assert float((vd / s - ref).abs().max()) <= 2e-5 * float(ref.abs().max())


def test_bn_prelu_bwd_bf16():
    """bf16 storage of y, the gradient source, du and dy (in place)."""
    N, T, C, padL, padR, pool_d = 2, 203, 64, 4, 5, 16
    Tp = T + padL + padR
    y = R(N * T * C, seed=24).to(torch.bfloat16)
    mean, invstd = R(C, seed=25, scale=0.1), R(C, seed=26).abs() + 0.5
    scale, shift, alpha = R(C, seed=27), R(C, seed=28), R(C, seed=29, scale=0.3)
    srcA = R(N * Tp * C, seed=30).to(torch.bfloat16)
    pool_T = T // pool_d
    pool = R(N * pool_T * C, seed=32)
    dst = torch.zeros(N * T * C, dtype=torch.bfloat16)
    S1, S2, dal = (torch.zeros(C, dtype=torch.float64) for _ in range(3))
    cpu, dev = run_both("pase_bn_prelu_bwd_reduce", [
        y, 1, T * C, N, T, C, mean, invstd, scale, shift, alpha, srcA, 1, Tp * C, C, padL, padR,
        None, 0, 0, 0, pool, pool_T * C, C, pool_d, pool_T, dst, T * C, S1, S2, dal, None],
        rtol=2.0 ** -7, atol=2e-5)
    du, s1, s2 = cpu[26], cpu[28], cpu[29]
    run_both("pase_bn_prelu_bwd_apply", [y, 1, T * C, N, T, C, mean, invstd, R(C, seed=33), s1, s2,
                                         float(N * T), du, du.clone(), None, 1, T * C,
                                         torch.zeros(C, dtype=torch.float64), None, None],
             rtol=2.0 ** -7, atol=2e-5, skip=(12,))


def test_cast_and_split_f16():
    x = R(100003, seed=41) * 5.0
    cpu, dev = run_both("pase_cast_bf16", [x, torch.zeros(100003, dtype=torch.bfloat16), 100003],
                        rtol=0, atol=0)
    assert torch.equal(cpu[1], dev[1].cpu())
    hi, lo = torch.zeros(100003, dtype=torch.float16), torch.zeros(100003, dtype=torch.float16)
    cpu, dev = run_both("pase_split_f16", [x, hi, lo, 100003, None, None], rtol=0, atol=0)
    assert torch.equal(cpu[1], dev[1].cpu()) and torch.equal(cpu[2], dev[2].cpu())
    v = cpu[1].float() + cpu[2].float() / 2048.0
    assert float((v - x).abs().max()) <= float(x.abs().max()) * 2.0 ** -21
    # scaled (gradient) form: tiny values are lifted into fp16's range by a power of two
    g = R(50000, seed=42) * 3e-7
    am = torch.zeros(2)
    cpu, dev = run_both("pase_absmax", [g, 50000, am], rtol=0, atol=0)
    assert float(cpu[2][0]) == float(g.abs().max())
    sc = torch.zeros(2)
    cpu, dev = run_both("pase_split_f16", [g, torch.zeros(50000, dtype=torch.float16),
                                           torch.zeros(50000, dtype=torch.float16), 50000,
                                           cpu[2], sc], rtol=0, atol=0)
    assert torch.equal(cpu[1], dev[1].cpu()) and torch.equal(cpu[2], dev[2].cpu())
    s = float(cpu[5][1])
    v = (cpu[1].float() + cpu[2].float() / 2048.0) / s
    assert 8192.0 <= float(g.abs().max()) * s <= 16384.0
    assert float((v - g).abs().max()) <= float(g.abs().max()) * 2.0 ** -21


def test_prelu_colsum_cast():
    rows, C = 333, 84
    u, dh, a = R(rows * 90, seed=34), R(rows * 88, seed=35), R(C, seed=36, scale=0.3)
    run_both("pase_prelu_fwd", [u, torch.zeros(rows * 96), a, rows, C, 90, 96])
    run_both("pase_prelu_bwd", [u, dh, a, torch.zeros(rows * 96), torch.zeros(C, dtype=torch.float64),
                                rows, C, 90, 88, 96])
    run_both("pase_colsum", [u, 90, rows, C, torch.zeros(C, dtype=torch.float64)])
    wide = R(7 * 9000, seed=60)
    run_both("pase_colsum", [wide, 9000, 7, 8999, torch.zeros(8999, dtype=torch.float64)])
    run_both("pase_cast_d2f", [R(100, seed=37).double(), torch.zeros(100), 100, 0.5])


def test_output_norm_kernels():
    N, T, C = 3, 37, 100
    y = R(N * T * C, seed=38)
    sc, sh = R(C, seed=39), R(C, seed=40)
    run_both("pase_out_affine_nct", [y, sc, sh, torch.zeros(N * C * T), torch.zeros(N * T * C), N, T, C])
    mean, invstd = R(C, seed=41, scale=0.1), R(C, seed=42).abs() + 0.5
    S1, S2 = torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    cpu, _ = run_both("pase_out_bwd_reduce", [R(N * C * T, seed=43), R(N * T * C, seed=44), y, mean,
                                              invstd, N, T, C, torch.zeros(N * T * C), S1, S2])
    run_both("pase_out_bwd_apply", [cpu[8], y, mean, invstd, invstd, cpu[9], cpu[10], float(N * T), 1,
                                    N * T, C])
    run_both("pase_nct_to_ntc", [R(N * C * T, seed=45), torch.zeros(N * T * 104), N, C, T, 104])
    run_both("pase_ntc_to_nct", [R(N * T * 104, seed=46), 104, torch.zeros(N * C * T), N, C, T])


@pytest.mark.parametrize("N,T,H", [(3, 23, 96), (2, 200, 512), (2, 16, 40), (1, 300, 64),
                                   (1, 500, 32), (1, 700, 32), (2, 1, 33)])
def test_qrnn_scan(N, T, H):
    """T <= 512: time-segmented scans (16-step segments, 16 / 24 / 32 segments per block);
    longer: the sequential kernels."""
    Y = R(N * T * 3 * H, seed=47)
    ldh = H + 32
    cpu, _ = run_both("pase_qrnn_scan_fwd", [Y, torch.zeros(N * T * ldh), ldh, torch.zeros(N * T * H),
                                             N, T, H], rtol=2e-4, atol=2e-5)
    run_both("pase_qrnn_scan_bwd", [Y, cpu[3], R(N * T * ldh, seed=48), ldh, torch.zeros(N * T * 3 * H),
                                    N, T, H], rtol=5e-4, atol=5e-5)


def test_losses():
    B, F, T, r = 2, 13, 21, 7
    ldp = F * r + 1
    pred, label = R(B * T * ldp, seed=49), R(B * F * T, seed=50)
    run_both("pase_ctx_mse_fwd", [pred, ldp, label, B, F, T, r, torch.zeros(1, dtype=torch.float64)])
    gs = torch.tensor([0.7])
    run_both("pase_ctx_mse_bwd", [pred, ldp, label, B, F, T, r, 0.01, gs, torch.zeros(B * T * ldp), ldp])
    run_both("pase_ctx_mse_fwd", [pred, ldp, label, B, F, T, 1, torch.zeros(1, dtype=torch.float64)])
    n = 5000
    p, t = R(n, seed=51), R(n, seed=52)
    run_both("pase_l1_fwd", [p, t, n, torch.zeros(1, dtype=torch.float64)])
    run_both("pase_l1_bwd", [p, t, n, 0.01, gs, torch.zeros(n)])
    run_both("pase_bce_pairs_fwd", [p * 3, n, n // 2, torch.zeros(1, dtype=torch.float64)])
    run_both("pase_bce_pairs_bwd", [p * 3, n, n // 2, 0.01, None, torch.zeros(n)])
    Bm, Tm, Cm = 4, 19, 96
    x = R(Bm * Tm * 100, seed=53)
    run_both("pase_time_mean_fwd", [x, 100, torch.zeros(Bm * Cm), Cm, Bm, Tm, Cm])
    run_both("pase_time_mean_bwd", [R(Bm * Cm, seed=54), Cm, R(Bm * Tm * 100, seed=55), 100, Bm, Tm, Cm, 1])
    run_both("pase_axpy", [p, t, n, 0.3])
    run_both("pase_scale_dev", [p, n, gs, 2.0])


def test_error_reporting():
    with pytest.raises(RuntimeError, match="multiples of 4"):
        _lib.call("pase_gemm_nt", torch.zeros(64).cuda(), 3, torch.zeros(64).cuda(), 4,
                  torch.zeros(64).cuda(), 4, 4, 4, 4, 1.0, None, 4, 4, 4, 1, None, None, 0)
    with pytest.raises(RuntimeError, match="CUDA device"):
        _lib.call("pase_axpy", torch.zeros(4), torch.zeros(4).cuda(), 4, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("tiled", [False, True])
def test_conv_w_batch_matches_per_layer_ops(tiled):
    """pase_conv_w_batch == the per-layer re-layouts (+ explicit-hi TF32 split), bit-exact;
    tiled: the shared-memory variants (ops 3..5)."""
    layers = [(64, 64, 20, 10), (128, 64, 11, 2), (128, 128, 11, 1)]
    layers += [(512, 256, 11, 2), (32, 8, 3, 1)] if tiled else [(24, 12, 5, 2)]
    nosplit = layers[-1][0]
    dev = torch.device("cuda")
    Ws = [R(co, ci, k, seed=3 + i).to(dev) for i, (co, ci, k, s) in enumerate(layers)]

    def table(rows, op):
        out, start, blocks = [], 0, 0
        for r in rows:
            out.append(r[:9] + [start, r[9], blocks])
            start += r[9]
            blocks += (r[4] // 32) * (r[5] // 8) if op == 1 else r[4]
        t = torch.tensor(out, dtype=torch.int64, device=dev).reshape(-1)
        return (t, blocks, op + 3) if tiled else (t, start, op)

    for op in (0, 1):
        rows, outs, his, los, refs = [], [], [], [], []
        for W, (co, ci, k, s) in zip(Ws, layers):
            taps = (k + s - 1) // s
            cnt = co * ci * k if op == 0 else s * ci * taps * co
            o, h, l = (torch.full((cnt,), 7.0, device=dev) for _ in range(3))
            split = (co != nosplit)                    # last job: no split requested
            rows.append([W.data_ptr(), o.data_ptr(), h.data_ptr() if split else 0,
                         l.data_ptr() if split else 0, co, ci, k, s, taps, cnt])
            ref = torch.empty(cnt, device=dev)
            if op == 0:
                _lib.call("pase_conv_w_to_fwd", W.reshape(-1), ref, co, ci, k)
            else:
                _lib.call("pase_conv_w_to_dgrad", W.reshape(-1), ref, co, ci, k, s, taps)
            rh, rl = torch.empty(cnt, device=dev), torch.empty(cnt, device=dev)
            _lib.call("pase_split_tf32", ref, rh, rl, cnt)
            outs.append(o)
            his.append(h if split else None)
            los.append(l if split else None)
            refs.append((ref, rh, rl))
        t, total, opc = table(rows, op)
        _lib.call("pase_conv_w_batch", t, len(rows), total, opc, None, 0)
        torch.cuda.synchronize()
        for o, h, l, (ref, rh, rl) in zip(outs, his, los, refs):
            assert torch.equal(o, ref)
            if h is not None:
                assert torch.equal(h, rh) and torch.equal(l, rl)

    # op 2: GEMM-layout gradients -> parameter layout, into one flat buffer
    rows, refs, off = [], [], 0
    srcs = [R(co, k, ci, seed=11 + i).to(dev) for i, (co, ci, k, s) in enumerate(layers)]
    for S, (co, ci, k, s) in zip(srcs, layers):
        cnt = co * ci * k
        rows.append([S.data_ptr(), off, 0, 0, co, ci, k, 1, 1, cnt])
        ref = torch.empty(cnt, device=dev)
        _lib.call("pase_conv_w_from_fwd", S.reshape(-1), ref, co, ci, k)
        refs.append((off, cnt, ref))
        off += cnt
    t, total, opc = table(rows, 2)
    flat = torch.zeros(off, device=dev)
    _lib.call("pase_conv_w_batch", t, len(rows), total, opc, flat, 0)
    torch.cuda.synchronize()
    for o, cnt, ref in refs:
        assert torch.equal(flat[o:o + cnt], ref)
