"""pase_tc_gemm_nt_plan on the CPU: how the NT GEMM of every tensor-core launch of the PASE+
training step (B=32, T=32000, 3xf16) covers its output on a 132-SM H100.  A launch whose
128-wide tiles fill R >= 1 rounds plus part of one more runs the first rows in at most R
rounds, and the rows left in one round of narrower tiles, when they fit one round."""
import os

import pytest

from pase_b200 import _lib

SMS = 132

# M, N, K of the step's pase_tc_gemm_nt launches in program order, and the tail tile width
# the plan picks (0: one launch)
STEP = [
    ("sinc fwd", 16128, 4096, 320, 0),
    ("block1 fwd", 102464, 64, 1280, 8),
    ("block2 fwd", 51360, 128, 704, 8),
    ("block3 fwd", 51520, 128, 1408, 8),
    ("block4 fwd", 25760, 256, 1408, 8),
    ("block5 fwd", 25920, 256, 2816, 16),
    ("block6 fwd", 12960, 512, 2816, 16),
    ("block7 fwd", 6560, 512, 5632, 0),
    ("qrnn fwd", 6432, 1536, 1024, 0),
    ("W+skips fwd", 6400, 256, 1920, 0),
    ("W+skips dgrad", 6400, 1920, 256, 0),
    ("qrnn dgrad", 6400, 1024, 1536, 8),
    ("block7 dgrad", 6720, 1024, 3072, 32),
    ("block6 dgrad", 13120, 512, 3072, 16),
    ("block5 dgrad", 26240, 256, 2816, 16),
    ("block4 dgrad", 25920, 256, 1536, 16),
    ("block3 dgrad", 51840, 128, 1408, 16),
    ("block2 dgrad", 51520, 128, 768, 8),
    ("block1 dgrad", 102496, 640, 128, 64),
]


@pytest.fixture(scope="module", autouse=True)
def library():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()


def _ceil(a, b):
    return -(-a // b)


@pytest.mark.parametrize("name,M,N,K,tail_bn", STEP, ids=[s[0] for s in STEP])
def test_step_plan(name, M, N, K, tail_bn):
    p = _lib.tc_gemm_nt_plan(M, N, SMS)
    bn = 64 if N <= 64 else 128
    assert p["bn"] == bn
    tiles = _ceil(M, 128) * _ceil(N, bn)
    rounds, left = divmod(tiles, SMS)
    assert p["tail_bn"] == tail_bn, p
    if tail_bn == 0:
        assert p["bulk_m"] == M and p["tail_pieces"] == 0
        # no tail only where there is no partial round after a whole one, or its rows do not
        # fit one round even in 8-wide tiles
        mb = rounds * SMS // _ceil(N, bn)
        assert rounds == 0 or left == 0 or (_ceil(M, 128) - mb) * _ceil(N, 8) > SMS
        return
    assert rounds >= 1 and left > 0
    bulk_m = p["bulk_m"]
    assert bulk_m % 128 == 0 and 0 < bulk_m < M
    assert bulk_m // 128 * _ceil(N, bn) <= rounds * SMS          # the bulk: at most R rounds
    pieces = _ceil(M - bulk_m, 128) * _ceil(N, tail_bn)
    assert p["tail_pieces"] == pieces <= SMS                     # the tail: one round
    assert tail_bn in (8, 16, 32, 64) and tail_bn < bn
    if tail_bn > 8:                                              # the narrowest that fits
        assert _ceil(M - bulk_m, 128) * _ceil(N, tail_bn // 2) > SMS


def test_launches_per_step():
    """14 of the step's 19 NT GEMMs run their last round in narrow tiles."""
    assert sum(_lib.tc_gemm_nt_plan(M, N, SMS)["tail_bn"] > 0 for _, M, N, _, _ in STEP) == 14


@pytest.mark.parametrize("M,N", [(128, 128), (300, 64), (132 * 128, 128), (132 * 128 * 2, 256)])
def test_whole_rounds_and_small_outputs_take_one_launch(M, N):
    p = _lib.tc_gemm_nt_plan(M, N, SMS)
    assert p["tail_bn"] == 0 and p["bulk_m"] == M


def test_bad_args():
    with pytest.raises(RuntimeError):
        _lib.tc_gemm_nt_plan(0, 128, SMS)
    with pytest.raises(RuntimeError):
        _lib.tc_gemm_nt_plan(128, 128, 0)
