"""BatchNorm column statistics of the wgmma NT GEMM (`colsum` / `colsumsq` of pase_tc_gemm_nt)
against float64 column sums of the kernel's own output, in the regimes the training step runs
them: the sinc layer's 4096 statistic columns (fold 64 x 64 channels, K = 320) over several row
groups whose last rows are partly masked by t_valid, with each CTA running several tiles; and
shapes whose last round runs as a second launch of narrow tiles (nt_plan), so the column sums
are the bulk's and the tail's added together.  The bound is the column-sum convention of the
BatchNorm kernels: 2^-16 of the sum of the terms' magnitudes.  Two runs at the sinc shape must
give equal fp32 pase_bn_finalize outputs."""
import pytest
import torch

from pase_b200 import _lib

pytestmark = pytest.mark.gpu

MODES = {"3xtf32": 1, "bf16": 2, "3xf16": 3}
# the sinc layer of the PASE+ step in 3xf16 at T = 32000 (16 groups of 504 folded rows, 500
# written), here 8 groups with t_valid cutting into the last written row
SINC = dict(N=4096, K=320, Rr=64, rows_in=504, t_valid=31990, rows_out=500, fold=64, groups=8)


def _randn(n, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return scale * torch.randn(n, generator=g, device="cuda")


def _operand(x, mode, weights):
    """(hi, lo) of x in GEMM mode `mode`, as the product builds them."""
    if mode == 2:
        return x.to(torch.bfloat16), None
    if mode == 3:
        hi = x.to(torch.float16)
        return hi, ((x - hi.float()) * 2048.0).to(torch.float16)
    lo = torch.empty_like(x)
    hi = torch.empty_like(x) if weights else None
    _lib.call("pase_split_tf32", x, hi, lo, x.numel())
    return (hi if weights else x), lo


def _gemm(mode, M, N, K, Rr, rows_in, t_valid, rows_out, fold, seed):
    """One pase_tc_gemm_nt call with statistics on seeded operands -> (C, colsum, colsumsq)."""
    a_rows = M + (K + Rr - 1) // Rr + 1
    (Ah, Al) = _operand(_randn(a_rows * Rr, seed), mode, False)
    (Bh, Bl) = _operand(_randn(N * K, seed + 1, 0.05), mode, True)
    bias = _randn(N, seed + 2)
    groups = -(-M // rows_in)
    C = torch.zeros(groups * rows_out * N, device="cuda")
    cs, cq = (torch.zeros(N, dtype=torch.float64, device="cuda") for _ in range(2))
    _lib.call("pase_tc_gemm_nt", Ah, Al, a_rows, Rr, Bh, Bl, K, C, N, M, N, K, 1.0, None, bias,
              rows_in, t_valid, rows_out, fold, cs, cq, 0, mode, 0)
    torch.cuda.synchronize()
    return C, cs, cq


def _check_stats(what, C, cs, cq, M, N, rows_in, t_valid, rows_out, fold):
    """colsum / colsumsq against float64 sums over the output elements the row map writes:
    rows u < min(rows_in, rows_out) of each group, columns n < (t_valid - u fold) N / fold."""
    groups = -(-M // rows_in)
    assert M == groups * rows_in
    u = torch.arange(rows_out, device="cuda")
    lim = ((t_valid - u * fold) * (N // fold)).clamp(0, N)
    lim = torch.where(u < rows_in, lim, torch.zeros_like(lim))
    mask = torch.arange(N, device="cuda")[None, :] < lim[:, None]
    y = C.view(groups, rows_out, N).double() * mask
    worst = 0.0
    for name, got, terms in (("colsum", cs, y), ("colsumsq", cq, y * y)):
        ref = terms.sum((0, 1))
        tol = 2.0 ** -16 * terms.abs().sum((0, 1))
        err = (got - ref).abs()
        assert bool((err <= tol).all()), "%s %s: %d/%d columns out of bound, worst err %.3e " \
            "tol %.3e" % (what, name, int((err > tol).sum()), N, float(err.max()),
                          float(tol[torch.argmax(err)]))
        worst = max(worst, float((err / tol.clamp_min(1e-300)).max()))
    print("%s: worst err / bound %.3g" % (what, worst))


@pytest.mark.parametrize("prec", list(MODES))
def test_sinc_statistics(prec):
    s = SINC
    M = s["groups"] * s["rows_in"]
    sms = _lib.device_info()["sms"]
    assert -(-M // 128) * (s["N"] // 128) > 2 * sms, "every CTA should run several tiles"
    # t_valid cuts into the last written row of each group
    last = s["t_valid"] - (s["rows_out"] - 1) * s["fold"]
    assert 0 < last < s["fold"] and s["rows_out"] < s["rows_in"]
    C, cs, cq = _gemm(MODES[prec], M, s["N"], s["K"], s["Rr"], s["rows_in"], s["t_valid"],
                      s["rows_out"], s["fold"], 11)
    _check_stats("sinc " + prec, C, cs, cq, M, s["N"], s["rows_in"], s["t_valid"],
                 s["rows_out"], s["fold"])


def test_sinc_statistics_finalize_reproducible():
    s = SINC
    M = s["groups"] * s["rows_in"]
    Cc = s["N"] // s["fold"]
    outs = []
    for _ in range(2):
        C, cs, cq = _gemm(3, M, s["N"], s["K"], s["Rr"], s["rows_in"], s["t_valid"],
                          s["rows_out"], s["fold"], 21)
        res = [torch.zeros(Cc, device="cuda") for _ in range(4)]
        rm, rv = torch.zeros(Cc, device="cuda"), torch.ones(Cc, device="cuda")
        _lib.call("pase_bn_finalize", cs, cq, Cc, s["fold"], float(s["groups"] * s["t_valid"]),
                  torch.ones(Cc, device="cuda"), torch.zeros(Cc, device="cuda"), rm, rv, 0.1,
                  1e-5, *res)
        torch.cuda.synchronize()
        outs.append((C, cs, cq, res + [rm, rv]))
    (C1, s1, q1, o1), (C2, s2, q2, o2) = outs
    assert torch.equal(C1, C2)
    for a, b in ((s1, s2), (q1, q2)):
        assert float((a - b).abs().max()) <= 1e-14 * float(a.abs().max())
    for a, b in zip(o1, o2):
        assert torch.equal(a, b)


# name, M, N, K, R, rows_in, t_valid, rows_out (fold 1), tail width at 132 SMs
TAIL_SHAPES = [
    ("block3_fwd", 51520, 128, 1408, 128, 1610, 1600, 1600, 8),
    ("block6_fwd", 12960, 512, 2816, 256, 405, 400, 400, 16),
    ("block7_dgrad", 6720, 1024, 3072, 512, 210, 200, 200, 32),
]


@pytest.mark.parametrize("prec", ["3xf16", "bf16"])
@pytest.mark.parametrize("name,M,N,K,Rr,rows_in,t_valid,rows_out,tail_bn", TAIL_SHAPES,
                         ids=[s[0] for s in TAIL_SHAPES])
def test_statistics_over_bulk_and_tail(name, M, N, K, Rr, rows_in, t_valid, rows_out, tail_bn,
                                       prec):
    sms = _lib.device_info()["sms"]
    plan = _lib.tc_gemm_nt_plan(M, N, sms)
    if sms == 132:
        assert plan["tail_bn"] == tail_bn, plan
    assert plan["tail_bn"] > 0, plan
    C, cs, cq = _gemm(MODES[prec], M, N, K, Rr, rows_in, t_valid, rows_out, 1, 31)
    _check_stats("%s %s" % (name, prec), C, cs, cq, M, N, rows_in, t_valid, rows_out, 1)
