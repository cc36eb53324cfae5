"""The wgmma NT GEMM's last round in narrow tiles (pase_tc_gemm_nt_plan): at shapes of the
B=32, T=32000 training step whose 128-wide tiles leave a partial last round, the rows of that
round run as a second launch of 128 x 8..64 tiles over the whole K.  A row's result must not
depend on the tile width, so every tail row must equal, bit for bit, the same row computed by
a call over the tail rows alone (fewer tiles than SMs: one launch of 128-wide tiles), and the
column statistics of the two launches must add up to those of the parts."""
import pytest
import torch

from pase_b200 import _lib

pytestmark = pytest.mark.gpu

# name, M, N, K, R (folded-row length of A), tail width at 132 SMs
SHAPES = [
    ("block3_fwd", 51520, 128, 1408, 128, 8),
    ("block6_fwd", 12960, 512, 2816, 256, 16),
    ("qrnn_dgrad", 6400, 1024, 1536, 1536, 8),
    ("block7_dgrad", 6720, 1024, 3072, 512, 32),
]
MODES = {"tf32": 0, "3xtf32": 1, "bf16": 2, "3xf16": 3}


def _randn(n, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return scale * torch.randn(n, generator=g, device="cuda")


def _operand(x, mode, weights):
    """(hi, lo) of x in GEMM mode `mode`, as the product builds them."""
    if mode == 0:
        return x, None
    if mode == 2:
        return x.to(torch.bfloat16), None
    if mode == 3:
        hi = x.to(torch.float16)
        return hi, ((x - hi.float()) * 2048.0).to(torch.float16)
    lo = torch.empty_like(x)
    hi = torch.empty_like(x) if weights else None
    _lib.call("pase_split_tf32", x, hi, lo, x.numel())
    return (hi if weights else x), lo


def _rows(t, row0, width):
    return None if t is None else t[row0 * width:]


def _gemm(A, a_rows, Rr, B, K, C, M, N, bias, alpha_dev, stats, acc, mode):
    (Ah, Al), (Bh, Bl) = A, B
    cs = torch.zeros(N, dtype=torch.float64, device="cuda") if stats else None
    cq = torch.zeros(N, dtype=torch.float64, device="cuda") if stats else None
    _lib.call("pase_tc_gemm_nt", Ah, Al, a_rows, Rr, Bh, Bl, K, C, N, M, N, K, 1.0, alpha_dev,
              bias, M, M, M, 1, cs, cq, acc, mode, 0)
    return cs, cq


@pytest.mark.parametrize("epilogue", ["stats", "accumulate"])
@pytest.mark.parametrize("prec", list(MODES))
@pytest.mark.parametrize("name,M,N,K,Rr,tail_bn", SHAPES, ids=[s[0] for s in SHAPES])
def test_tail_rows_equal_a_call_over_them_alone(name, M, N, K, Rr, tail_bn, prec, epilogue):
    mode = MODES[prec]
    sms = _lib.device_info()["sms"]
    plan = _lib.tc_gemm_nt_plan(M, N, sms)
    tiles = -(-M // 128) * -(-N // plan["bn"])
    rounds = tiles // sms
    if sms == 132:
        assert plan["tail_bn"] == tail_bn, plan
    assert plan["tail_bn"] > 0 and rounds >= 1, plan
    bulk_m = plan["bulk_m"]
    assert bulk_m % 128 == 0 and 0 < bulk_m < M
    assert bulk_m // 128 * -(-N // plan["bn"]) <= rounds * sms
    tail_m = M - bulk_m
    assert plan["tail_pieces"] == -(-tail_m // 128) * -(-N // tail_bn) <= sms
    # over the tail rows alone: fewer tiles than SMs, one launch of the plain tiles
    assert _lib.tc_gemm_nt_plan(tail_m, N, sms)["tail_bn"] == 0

    a_rows = M + (K + Rr - 1) // Rr + 1
    x = _randn(a_rows * Rr, 1)
    w = _randn(N * K, 2, scale=0.05)
    A, B = _operand(x, mode, False), _operand(w, mode, True)
    bias = _randn(N, 3)
    alpha_dev = torch.tensor([0.75], device="cuda")
    stats, acc = epilogue == "stats", int(epilogue == "accumulate")
    C0 = _randn(M * N, 4) if acc else torch.zeros(M * N, device="cuda")

    C = C0.clone()
    cs, cq = _gemm(A, a_rows, Rr, B, K, C, M, N, bias, alpha_dev, stats, acc, mode)
    Ct = C0[bulk_m * N:].clone()
    At = tuple(_rows(t, bulk_m, Rr) for t in A)
    ts, tq = _gemm(At, a_rows - bulk_m, Rr, B, K, Ct, tail_m, N, bias, alpha_dev, stats, acc,
                   mode)
    torch.cuda.synchronize()
    tail = C[bulk_m * N:]
    bad = int((tail != Ct).sum())
    assert bad == 0, "%s %s: %d tail elements differ, max %.3e" % (
        name, prec, bad, float((tail - Ct).abs().max()))
    assert bool(torch.isfinite(C).all())
    if acc:     # the bulk rows too received exactly one write
        Cb = C0[:bulk_m * N].clone()
        _gemm(A, a_rows, Rr, B, K, Cb, bulk_m, N, bias, alpha_dev, False, 1, mode)
        torch.cuda.synchronize()
        assert torch.equal(C[:bulk_m * N], Cb)
    if stats:
        Cb = torch.zeros(bulk_m * N, device="cuda")
        bs, bq = _gemm(A, a_rows, Rr, B, K, Cb, bulk_m, N, bias, alpha_dev, True, 0, mode)
        torch.cuda.synchronize()
        assert torch.equal(C[:bulk_m * N], Cb)
        for full, part_b, part_t in ((cs, bs, ts), (cq, bq, tq)):
            ref = part_b + part_t
            lim = 1e-12 * float(ref.abs().max())
            assert float((full - ref).abs().max()) <= lim
