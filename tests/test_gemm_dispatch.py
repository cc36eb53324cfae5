"""pase_b200.gemm on the CPU: the tensor-core eligibility rule against the preconditions of the
tensor-core entry points (tests/emul/core.py asserts the PASE_CHECK_ARG checks of
csrc/gemm_tc.cu), the kernel each dispatcher picks, and the refusal of operands that exist only
in a 16-bit format when the shape is outside the tensor-core path."""
import itertools

import pytest
import torch

import emul
import pase_b200.ops as ops
from pase_b200 import gemm

TC_PRECISIONS = [n for n, p in gemm.PRECISIONS.items() if p.tc]


@pytest.fixture()
def launches(monkeypatch):
    names = []

    def record(name, *a):
        names.append(name)
        return emul.call(name, *a)
    monkeypatch.setattr(ops, "call", record)
    return names


def _accepts(name, *args):
    try:
        emul.call(name, *args)
    except AssertionError:
        return False
    return True


def _rand(n, seed):
    return torch.randn(n, generator=torch.Generator().manual_seed(seed))


def test_precision_table():
    assert sorted(gemm.PRECISIONS) == ["3xf16", "3xtf32", "bf16", "fp32", "tf32"]
    for name, p in gemm.PRECISIONS.items():
        assert p.name == name and p.eb * p.esz == 128
        assert p.sinc_fold == (p.eb if p.tc else 4)
    assert [gemm.PRECISIONS[n].mode for n in ("tf32", "3xtf32", "bf16", "3xf16")] == [0, 1, 2, 3]
    assert not gemm.nt_ok(gemm.PRECISIONS["fp32"], 64, 64, 64)
    assert not gemm.tn_ok(gemm.PRECISIONS["fp32"], 64, 64, 64, 64)


@pytest.mark.parametrize("prec", TC_PRECISIONS)
def test_nt_rule_matches_the_entry_point(prec, launches):
    p = gemm.PRECISIONS[prec]
    M, N = 8, 8
    for R, K, dl in itertools.product((16, 32, 48, 64, 96, 128), (4, 6, 8, 12, 24, 40, 72),
                                      (-4, 0, 2, 4, 8)):
        ldb = K + dl
        if ldb <= 0:
            continue
        a_n = (M + (K + R - 1) // R + 1) * R
        A, B = _rand(a_n, 1), _rand(N * ldb, 2)
        a, b = gemm.to_operand(p, A, a_n), gemm.to_operand(p, B, B.numel(), "weight")
        args = (a.hi, a.lo, a_n // R, R, b.hi, b.lo, ldb, torch.zeros(M * N), N, M, N, K, 1.0,
                None, None, M, M, M, 1, None, None, 0, p.mode, 0)
        ok = gemm.nt_ok(p, R, K, ldb)
        assert ok == _accepts("pase_tc_gemm_nt", *args), (prec, R, K, ldb)
        launches.clear()
        if ldb >= K:
            gemm.nt(p, A, R, a_n, B, ldb, torch.zeros(M * N), N, M, N, K)
            assert launches[-1] == ("pase_tc_gemm_nt" if ok else "pase_gemm_nt"), (R, K, ldb)


@pytest.mark.parametrize("prec", TC_PRECISIONS)
def test_tn_rule_matches_the_entry_point(prec, launches):
    p = gemm.PRECISIONS[prec]
    rows = 8
    for R, lda, I, J in itertools.product((16, 32, 48, 64, 128), (6, 8, 12, 16, 64), (4, 6, 8),
                                          (8, 32, 64, 96)):
        if I > lda:
            continue
        a_n, b_n = rows * lda, (rows + (J + R - 1) // R) * R
        A, B = _rand(a_n, 3), _rand(b_n, 4)
        a, b = gemm.to_operand(p, A, a_n, "grad"), gemm.to_operand(p, B, b_n)
        args = (a.hi, a.lo, lda, rows, 0, b.hi, b.lo, R, rows, b_n // R, torch.zeros(I * J), J,
                I, J, 1, rows, 1.0, a.alpha, 0, p.mode)
        ok = gemm.tn_ok(p, lda, R, I, J)
        assert ok == _accepts("pase_tc_gemm_tn", *args), (prec, R, lda, I, J)
        launches.clear()
        gemm.tn(p, A, lda, a_n, B, R, b_n, torch.zeros(I * J), J, I, J, rows)
        assert launches[-1] == ("pase_tc_gemm_tn" if ok else "pase_gemm_tn"), (R, lda, I, J)


@pytest.mark.parametrize("prec", ["bf16", "3xf16"])
def test_16bit_only_operand_outside_the_tensor_core_path_is_refused(prec, launches):
    p = gemm.PRECISIONS[prec]
    C = torch.zeros(64)
    only16 = torch.zeros(40 * 8, dtype=p.dtype)          # written by its producer in p's format
    with pytest.raises(NotImplementedError, match="outside the tensor-core path"):
        gemm.nt(p, only16, 40, only16.numel(), _rand(8 * 40, 5), 40, C, 8, 8, 8, 40)
    with pytest.raises(NotImplementedError, match="outside the tensor-core path"):
        gemm.nt(p, None, 40, 8 * 40, _rand(8 * 40, 5), 40, C, 8, 8, 8, 40,
                a_op=gemm.Operand(only16))
    with pytest.raises(NotImplementedError, match="weight-gradient GEMM shape"):
        gemm.tn(p, _rand(8 * 8, 6), 8, 64, only16, 40, only16.numel(), C, 8, 8, 8, 8)
    assert launches == []
    # fp32 operands of a shape outside the tensor-core path take the FFMA kernel
    gemm.nt(p, _rand(8 * 40, 7), 40, 8 * 40, _rand(8 * 40, 5), 40, C, 8, 8, 8, 40)
    assert launches == ["pase_gemm_nt"]
