"""GEMM precision and dispatch for the encoder, the worker heads and the decoder: the five
precisions, their operand formats, and which kernel runs a GEMM (pase_tc_gemm_* on the tensor
cores or pase_gemm_* on FFMA).  Numerics of each precision: DESIGN.md section 5."""
from typing import NamedTuple, Optional

import torch

from . import ops

FMT_F32, FMT_BF16, FMT_F16X2 = 0, 1, 2         # operand storage formats of the C-ABI


class Precision(NamedTuple):
    name: str
    mode: Optional[int]       # `mode` of pase_tc_gemm_*; None: the fp32 FFMA kernels
    dtype: torch.dtype        # element type of the operand buffers
    fmt: int                  # FMT_* code of the operand format
    split: bool               # operands are (hi, lo) pairs
    act_bf16: bool            # raw conv outputs and activation gradients stored in bf16

    tc = property(lambda self: self.mode is not None)
    esz = property(lambda self: self.dtype.itemsize)
    eb = property(lambda self: 128 // self.esz)                  # elements per 128-byte row
    # fp32 / tf32 GEMMs read the fp32 tensors themselves: no operand buffers
    reads_fp32 = property(lambda self: self.fmt == FMT_F32 and not self.split)
    # polyphase fold of the sinc layer: one 128-byte row on the tensor cores
    sinc_fold = property(lambda self: self.eb if self.tc else 4)


PRECISIONS = {p.name: p for p in (
    Precision("fp32", None, torch.float32, FMT_F32, False, False),
    Precision("3xtf32", 1, torch.float32, FMT_F32, True, False),
    Precision("tf32", 0, torch.float32, FMT_F32, False, False),
    Precision("bf16", 2, torch.bfloat16, FMT_BF16, False, True),
    Precision("3xf16", 3, torch.float16, FMT_F16X2, True, False),
)}


class Operand(object):
    """A GEMM operand in a precision's format.  hi / lo: as pase_tc_gemm_* takes them (lo None
    outside the split formats); alpha: device {1/s, s} of a power-of-two scaled 3xF16 gradient,
    amax: the bound s is derived from; src: the fp32 tensor it is converted from (None when its
    producer writes the operand format directly)."""
    __slots__ = ("hi", "lo", "alpha", "amax", "src")

    def __init__(self, hi, lo=None, alpha=None, amax=None, src=None):
        self.hi, self.lo, self.alpha, self.amax, self.src = hi, lo, alpha, amax, src


def operand_buffers(p, n, device, kind="act", src=None, new=torch.empty):
    """The Operand of n elements of kind 'act' | 'weight' | 'grad' in p's format, allocated with
    `new` and nothing launched.  fp32 / tf32 operands, and the hi part of a 3xTF32 activation
    (the tensor cores truncate it), are `src` itself."""
    if p.reads_fp32:
        return Operand(src, src=src)
    buf = lambda: new(n, dtype=p.dtype, device=device)
    scaled = p.fmt == FMT_F16X2 and kind == "grad"
    f2 = lambda: new(2, dtype=torch.float32, device=device) if scaled else None
    hi = src if p.fmt == FMT_F32 and kind != "weight" else buf()
    return Operand(hi, buf() if p.split else None, f2(), f2(), src)


def convert(p, op, n, kind="act"):
    """Launch the conversion of op.src[:n] into op's buffers and return op.  3xtf32: activations
    lo = rn(x - trunc(x)), weights hi = rn(x), lo = rn(x - hi); bf16: a bf16 copy; 3xf16: the
    fp16 (hi, lo') pair, gradients scaled by a power of two."""
    if p.fmt == FMT_F32 and p.split:
        ops.call("pase_split_tf32", op.src, op.hi if kind == "weight" else None, op.lo, n)
    elif p.fmt == FMT_BF16:
        ops.call("pase_cast_bf16", op.src, op.hi, n)
    elif p.fmt == FMT_F16X2:
        if op.amax is not None:
            op.amax.zero_()
            ops.call("pase_absmax", op.src, n, op.amax)
        ops.call("pase_split_f16", op.src, op.hi, op.lo, n, op.amax, op.alpha)
    return op


def to_operand(p, src, n, kind="act"):
    """fp32 src[:n] converted into new buffers of p's format."""
    return convert(p, operand_buffers(p, n, src.device, kind, src), n, kind)


# The shapes the tensor-core entry points accept: the PASE_CHECK_ARG lines of csrc/gemm_tc.cu
# (R: the row length of the operand read in 128-byte boxes, A of NT and B of TN)
#   pase_tc_gemm_nt:  R >= eb && (R % eb) == 0;
#                     (K * esz) % 16 == 0 && (ldb * esz) % 16 == 0 && ldb >= K
#   pase_tc_gemm_tn:  R >= eb && (R % eb) == 0 && (lda * esz) % 16 == 0 && (I % 4) == 0 &&
#                     (J % eb) == 0
# Their 16-byte operand alignment holds for every buffer handed to them.
def nt_ok(p, lda, K, ldb):
    return p.tc and lda >= p.eb and lda % p.eb == 0 and (K * p.esz) % 16 == 0 and \
        (ldb * p.esz) % 16 == 0 and ldb >= K


def tn_ok(p, lda, ldb, I, J):
    return p.tc and ldb >= p.eb and ldb % p.eb == 0 and (lda * p.esz) % 16 == 0 and \
        I % 4 == 0 and J % p.eb == 0


def _ffma_operands(p, what, *tensors):
    """The FFMA kernels read fp32: an operand that exists only in a 16-bit format is refused."""
    if any(t is None or t.dtype != torch.float32 for t in tensors):
        raise NotImplementedError("precision %r: %s outside the tensor-core path" % (p.name, what))


def _tc_operand(op, p, t, n, kind):
    op = op() if callable(op) else op
    return op if op is not None else to_operand(p, t, n, kind)


def nt(p, A, lda, a_n, B, ldb, C, ldc, M, N, K, alpha=1.0, bias=None, rows_in=None,
       t_valid=None, rows_out=None, fold=1, cs=None, cq=None, acc=0, a_kind="act", a_op=None,
       b_op=None):
    """C[map(m), n] (+)= alpha sum_k A[m*lda + k] B[n*ldb + k] + bias[n] in precision p; row map
    and column statistics as in pase_gemm_nt.  A (a_n elements) / B: the fp32 tensors the FFMA
    kernel reads (None, or the 16-bit buffer, for an operand that exists only in that format);
    the tensor-core path converts them unless a_op / b_op give the Operand (or a function
    returning it)."""
    if rows_in is None:
        rows_in = t_valid = rows_out = M
    if not nt_ok(p, lda, K, ldb):
        _ffma_operands(p, "GEMM shape (lda=%d K=%d)" % (lda, K), A, B)
        return ops.call("pase_gemm_nt", A, lda, B, ldb, C, ldc, M, N, K, alpha, bias,
                        rows_in, t_valid, rows_out, fold, cs, cq, acc)
    a = _tc_operand(a_op, p, A, a_n, a_kind)
    b = _tc_operand(b_op, p, B, None if B is None else B.numel(), "weight")
    return ops.call("pase_tc_gemm_nt", a.hi, a.lo, a_n // lda, lda, b.hi, b.lo, ldb, C, ldc,
                    M, N, K, alpha, a.alpha, bias, rows_in, t_valid, rows_out, fold, cs, cq, acc,
                    p.mode, 1 if C.dtype == torch.bfloat16 else 0)


def nt_var(p, A, lda, a_n, B, ldb, C, ldc, M, N, K, bias, tab, n, fold, a_op=None, b_op=None,
           cs=None, cq=None):
    """nt over a packed variable-length batch: the row map is the device table `tab` of n
    utterances (pase_gemm_nt_var); operands as for nt.  cs / cq (train mode): the BatchNorm
    column statistics of the stored elements (pase_gemm_nt_var_stats)."""
    stats = () if cs is None else (cs, cq)
    suffix = "" if cs is None else "_stats"
    if not nt_ok(p, lda, K, ldb):
        _ffma_operands(p, "GEMM shape (lda=%d K=%d)" % (lda, K), A, B)
        return ops.call("pase_gemm_nt_var" + suffix, A, lda, B, ldb, C, ldc, M, N, K, bias, tab,
                        n, fold, *stats)
    a = _tc_operand(a_op, p, A, a_n, "act")
    b = _tc_operand(b_op, p, B, None if B is None else B.numel(), "weight")
    return ops.call("pase_tc_gemm_nt_var" + suffix, a.hi, a.lo, a_n // lda, lda, b.hi, b.lo, ldb,
                    C, ldc, M, N, K, bias, tab, n, fold, *stats, p.mode,
                    1 if C.dtype == torch.bfloat16 else 0)


def tn(p, A, lda, a_n, B, ldb, b_n, C, ldc, I, J, rows, groups=1, pitchA=None, offA=0,
       pitchB=None, alpha=1.0, acc=0, a_kind="grad", a_op=None, b_op=None):
    """C[i, j] (+)= alpha sum_r A[rowA(r)*lda + i] B[rowB(r)*ldb + j] over `groups` x `rows` rows
    (group pitches pitchA / pitchB rows, A starting offA rows into its group) in precision p.
    Operands as for nt."""
    pitchA = rows if pitchA is None else pitchA
    pitchB = rows if pitchB is None else pitchB
    if not tn_ok(p, lda, ldb, I, J):
        _ffma_operands(p, "weight-gradient GEMM shape (lda=%d ldb=%d I=%d J=%d)"
                       % (lda, ldb, I, J), A, B)
        return ops.call("pase_gemm_tn", A, lda, pitchA, offA, B, ldb, pitchB, 0, C, ldc, I, J,
                        groups, rows, alpha, acc)
    a = _tc_operand(a_op, p, A, a_n, a_kind)
    b = _tc_operand(b_op, p, B, b_n, "act")
    return ops.call("pase_tc_gemm_tn", a.hi, a.lo, lda, pitchA, offA, b.hi, b.lo, ldb, pitchB,
                    b_n // ldb, C, ldc, I, J, groups, rows, alpha, a.alpha, acc, p.mode)
