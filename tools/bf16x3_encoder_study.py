#!/usr/bin/env python
"""CPU study: would the whole PASE+ encoder still meet the parity bar if every tensor-core
GEMM used three bf16 products of a two-term bf16 operand split (a1 b1 + a1 b2 + a2 b1)
instead of 3xTF32?  Runs the host orchestration of pase_b200 with the torch emulation of the
kernels (tests/emul/), swaps the product model of the two GEMM entry points, and
compares forward outputs and gradients with the golden vectors of the unmodified reference.
Measurement helper for the next round's kernel work; not part of the library or the tests.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, _p)

import emul                                                  # noqa: E402
from helpers import load_golden, resolve_cfg, fill_state_dict, seeded_randn, rel_l2   # noqa: E402
from detweights import sample_view                            # noqa: E402
import pase_b200.ops as ops                                  # noqa: E402
from pase_b200.frontend import WaveFe                        # noqa: E402
from test_host_emulated import run_encoder_cpu               # noqa: E402


def bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


def split2(x):
    x1 = bf16(x)
    return x1, bf16(x - x1)


class Bf16x3(object):
    """Product model: exact fp32 products of bf16 factors, three of the four cross terms."""

    @staticmethod
    def nt(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, alpha, bias, rows_in, t_valid,
           rows_out, fold, colsum, colsumsq, accumulate, mode, terms=None):
        terms = terms or _bf16_terms
        need = M * R + K
        a = torch.zeros(need)
        lim = min(a_rows * R, Ahi.numel(), need)
        a[:lim] = Ahi[:lim]                                  # activations: the raw fp32 array
        b = Bhi[:N * ldb].clone()
        if Blo is not None:
            b += emul.core._like(Blo, Bhi)[:N * ldb]         # weights: hi + lo = the fp32 value
        first = True
        for x, y in terms(a, b):
            emul.core.pase_gemm_nt(x, R, y, ldb, C, ldc, M, N, K, alpha, bias if first else None,
                                   rows_in, t_valid, rows_out, fold, None, None,
                                   accumulate if first else 1)
            first = False
        if colsum is not None:                               # statistics of the final values
            m = torch.arange(M)
            g, u = m // rows_in, m % rows_in
            keep = (u * fold) < t_valid
            cpf = N // fold
            valid = (u[keep][:, None] * fold + (torch.arange(N) // cpf)[None, :]) < t_valid
            orow = (g * rows_out + u)[keep]
            Cv = emul.core._as(C, (int(orow.max()) + 1, N), (ldc, 1))[orow]
            ov = torch.where(valid, Cv, torch.zeros_like(Cv)).double()
            colsum[:N] += ov.sum(0)
            colsumsq[:N] += (ov * ov).sum(0)

    @staticmethod
    def tn(Ahi, Alo, lda, pitchA, offA, Bhi, Blo, R, pitchB, b_rows_total, C, ldc, I, J, groups,
           rows_per_group, alpha, accumulate, mode, terms=None):
        terms = terms or _bf16_terms
        needB = ((groups - 1) * pitchB + rows_per_group) * R + J
        b = torch.zeros(max(needB, Bhi.numel()))
        lim = min(b_rows_total * R, Bhi.numel())
        b[:lim] = Bhi[:lim]
        first = True
        for x, y in terms(Ahi.clone(), b):
            emul.core.pase_gemm_tn(x, lda, pitchA, offA, y, R, pitchB, 0, C, ldc, I, J, groups,
                                   rows_per_group, alpha, accumulate if first else 1)
            first = False


def _tf32_terms(a, b):
    """(x, y) factor pairs of the mixed scheme: TF32 main product + two bf16 corrections."""
    ah, bh = emul.core._tf32_trunc(a), emul.core._tf32_rn(b)
    return ((ah, bh), (bf16(a - ah), bf16(b)), (bf16(a), bf16(b - bh)))


class Mixed(object):
    """trunc_tf32(a) rn_tf32(b) + bf16(a - a_hi) bf16(b) + bf16(a) bf16(b - b_hi)."""

    @staticmethod
    def nt(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, alpha, bias, rows_in, t_valid,
           rows_out, fold, colsum, colsumsq, accumulate, mode):
        Bf16x3.nt(Ahi, Alo, a_rows, R, Bhi, Blo, ldb, C, ldc, M, N, K, alpha, bias, rows_in,
                  t_valid, rows_out, fold, colsum, colsumsq, accumulate, mode, terms=_tf32_terms)

    @staticmethod
    def tn(Ahi, Alo, lda, pitchA, offA, Bhi, Blo, R, pitchB, b_rows_total, C, ldc, I, J, groups,
           rows_per_group, alpha, accumulate, mode):
        Bf16x3.tn(Ahi, Alo, lda, pitchA, offA, Bhi, Blo, R, pitchB, b_rows_total, C, ldc, I, J,
                  groups, rows_per_group, alpha, accumulate, mode, terms=_tf32_terms)


def _bf16_terms(a, b):
    a1, a2 = split2(a)
    b1, b2 = split2(b)
    return ((a1, b1), (a1, b2), (a2, b1))


def run(name, model_fns):
    gold, meta = load_golden(name)
    cfg = resolve_cfg(meta["cfg"])
    model = WaveFe(**cfg)
    model.precision = "3xtf32"
    model.load_state_dict(fill_state_dict(model.state_dict(), meta["seed"]))
    model.train(meta["training"])
    x = seeded_randn((meta["N"], 1, meta["T"]), meta["seed"] + 1, 0.5)
    saved = (emul.core.pase_tc_gemm_nt, emul.core.pase_tc_gemm_tn)
    if model_fns is not None:
        emul.core.pase_tc_gemm_nt, emul.core.pase_tc_gemm_tn = model_fns
    real = ops.call
    ops.call = emul.call
    try:
        y, _ = run_encoder_cpu(model, x)
        cot = seeded_randn(tuple(y.shape), meta["seed"] + 2)
        (y * cot).sum().backward()
    finally:
        ops.call = real
        emul.core.pase_tc_gemm_nt, emul.core.pase_tc_gemm_tn = saved
    yg = gold["y"]
    err = (y.detach() - yg).abs()
    worst = float((err / (1e-5 + 1e-3 * yg.abs())).max())    # <= 1 meets rtol 1e-3 / atol 1e-5
    gl2 = []
    for k, p in model.named_parameters():
        if k.endswith("conv.bias") or k == "W.bias":          # analytically zero under BN
            continue
        if "grad/" + k in gold:
            gl2.append((rel_l2(p.grad, gold["grad/" + k]), k))
        elif "gsample/" + k in gold:
            gl2.append((rel_l2(sample_view(p.grad.detach()), gold["gsample/" + k]), k))
    gl2.sort(reverse=True)
    return float(err.max()), worst, rel_l2(y.detach(), yg), gl2[:2]


if __name__ == "__main__":
    for name in ("enc_pasep_train_3200", "enc_pasep_train_4001", "enc_pase_train_2400"):
        for label, fns in (("3xtf32 (today)", None), ("tf32+2bf16", (Mixed.nt, Mixed.tn)),
                           ("3xbf16", (Bf16x3.nt, Bf16x3.tn))):
            mx, worst, l2, g = run(name, fns)
            print("%-22s %-15s fwd max err %.2e  err/tol %.3f  rel-L2 %.2e  worst grad rel-L2 %s"
                  % (name, label, mx, worst, l2,
                     ", ".join("%.2e (%s)" % (v, k) for v, k in g)))
