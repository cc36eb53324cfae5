"""The packed (*_var) and windowed (*_carry_var, pase_out_place_var, pase_out_bwd_gather_crop,
pase_reflect_fold_wave_acc, pase_stream_gather) entry points, one at a time, against a float64
reference computed with torch from exactly the operands each kernel reads, and, where the header
promises it, bit for bit against the uniform kernel run as a B=1 call on the same utterance.

Tables come from the product's builders where one exists (encoder.packed_grad_layout on a
PackedGradPlan for PASE+), with gaps added between utterances' outputs, and are hand-built for
the edges the builders rarely produce (T' = 1, windows of one recording, a boundary inside the
partial last round of the tensor-core GEMM).  Length lists: the encoder's minimum (471 samples)
with utterances of exactly 512 and 513 output frames (found with frame_counts), 48 seeded
lengths in 471..48000 in non-sorted order, and a single utterance.

Memory: gaps between utterances, slack rows and columns hold the 2^100 sentinel (65504 in fp16)
where a kernel must not read, or a guard value where it must not write; every guard is checked
unchanged after the call, so a store outside the contract fails even where a later kernel would
overwrite it.

Bounds (u = 2^-24) are those of the uniform kernels' tests, imported from them:
  GEMMs: the exact products of the operands as the tensor core reads them (emul.core._operand),
    accumulated in float64; error within 2 K u sum|a b| + 2^-20 sum|a b| (the 3x modes drop the
    lo x lo term) + 1 ulp of the bias add; bf16 output one more bf16 rounding.  colsum and
    colsumsq within 2^-16 of the sum of magnitudes of the stored values, against float64 sums
    of exactly the values the kernel stored.
  QRNN: the kappa = 32 bound of test_qrnn_sinc_out_gpu (qrnn_fwd_checks / qrnn_bwd_checks).
  BatchNorm/PReLU: dy within 2^-20 |gamma invstd| (|du| + |S1/M| + |xhat| |S2/M|), sums within
    2^-16 of the sum of the terms' magnitudes (test_bn_prelu_gpu).
  Output layer: one fmaf within 1 ulp; time means within 1e-6 max_t |h| (DESIGN.md section 11);
    S1 / S2 within 2^-16; gathers exact.
  Waveform pad exact (fp32, bf16 rounding, fp16 pair split exact); fold within 2u of the sum of
    the magnitudes of the (at most three) terms of each sample, and pad / fold adjoint in
    float64.
Each case prints its worst error as a fraction of its bound.  tests/test_packed_kernels.py runs
the same cases through the fp32 emulations on the CPU."""
import numpy as np
import pytest
import torch

import emul
from pase_b200 import _lib
from pase_b200 import encoder as E
from test_qrnn_sinc_out_gpu import (GUARD, K_QRNN, SENT, U, Qrnn, _check_all, _full, _report,
                                    _ulp32, _within, qrnn_bwd_checks, qrnn_fwd_checks)
from test_tc_gemm_gpu import _operands, _poison

pytestmark = pytest.mark.gpu

MAX_GRID_Y = 65535
F16_SENT = 65504.0
_cache = {}


# ---- shared helpers ----
def _call(dev, name, *args):
    """The CUDA kernel on a CUDA device, the fp32 torch emulation on the CPU."""
    if torch.device(dev).type == "cuda":
        _lib.call(name, *args)
        torch.cuda.synchronize()
    else:
        emul.call(name, *args)


def _gpu(dev):
    return torch.device(dev).type == "cuda"


def _i32(rows, dev):
    return torch.tensor(np.asarray(rows, dtype=np.int64).reshape(-1), dtype=torch.int32,
                        device=dev)


def _guard_mask(n, spans, dev):
    """Bool (n,): True outside every [a, b) of spans."""
    keep = torch.ones(int(n), dtype=torch.bool, device=dev)
    for a, b in spans:
        keep[int(a):int(b)] = False
    return keep


def _unchanged(what, buf, spans, value):
    rest = buf[_guard_mask(buf.numel(), spans, buf.device)]
    assert bool((rest == value).all()), "%s: written outside its contract" % what


def pasep_cfg():
    if "cfg" not in _cache:
        from helpers import resolve_cfg
        from pase_b200 import wf_builder
        _cache["cfg"] = wf_builder(resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    return _cache["cfg"]


def length_with_frames(cfg, want):
    """The shortest waveform whose encoder output has exactly `want` frames."""
    lo, hi = E.min_length(cfg), 1 << 24
    while lo < hi:
        mid = (lo + hi) // 2
        if E.frame_counts(cfg, mid)[-1] >= want:
            hi = mid
        else:
            lo = mid + 1
    assert E.frame_counts(cfg, lo)[-1] == want
    return lo


def length_lists(cfg):
    """{name: lengths}: the minimum with 512- and 513-frame utterances, 48 seeded lengths in
    471..48000 in non-sorted order, and a single utterance."""
    m = E.min_length(cfg)
    assert m == 471
    L512, L513 = length_with_frames(cfg, 512), length_with_frames(cfg, 513)
    rng = np.random.default_rng(48)
    seeded = [int(v) for v in rng.integers(m, 48001, size=48)]
    seeded[5], seeded[17] = m, 48000
    assert seeded != sorted(seeded)
    return {"edges": [m, L512, 3000, L513, m], "seeded48": seeded, "single": [17000]}


def product_layout(lengths, prec="fp32"):
    """The host table and sections encoder.packed_grad_layout uploads for these lengths, on a
    small-capacity PackedGradPlan for PASE+ (meta device: nothing is allocated)."""
    cfg = pasep_cfg()
    plan = E.PackedGradPlan(cfg, max(sum(lengths), 1 << 16), torch.device("meta"), prec)
    geoms = E.utterance_geometry(cfg, lengths, plan.precision.sinc_fold)
    host, sec, sz = E.packed_grad_layout(plan, lengths, geoms)
    return plan, geoms, host.numpy().astype(np.int64), sec, sz


# ================================ row-mapped GEMMs ================================
def _var_rows(tab, n):
    t = np.asarray(tab, dtype=np.int64)
    return t[:n + 1], t[n + 1:2 * n + 1], t[2 * n + 1:3 * n + 1]


def _stored_mask(P, t_valid, N, fold, dev):
    u = torch.arange(P, device=dev)[:, None]
    n = torch.arange(N, device=dev)[None, :]
    return u * fold + n // (N // fold) < t_valid


class VarGemm(object):
    """One packed NT GEMM: operand rows of every utterance, weights, a var_tab with gaps of
    `gap` output rows between utterances and `slack` GEMM rows past row0[nvar]."""

    def __init__(self, row0, t_valid, P_out, R, K, N, fold, mode, dev, gap=3, slack=37,
                 c_bf16=0, ldc=None, bias=True, seed=0):
        self.dev, self.R, self.K, self.N, self.fold, self.mode = dev, R, K, N, fold, mode
        self.c_bf16 = c_bf16
        n = len(t_valid)
        self.n = n
        self.row0 = np.asarray(row0, np.int64)
        self.t_valid = np.asarray(t_valid, np.int64)
        self.M = int(self.row0[-1]) + slack
        self.P = np.diff(self.row0)
        self.orow0 = np.concatenate([[0], np.cumsum(np.asarray(P_out) + gap)])[:n]
        self.ldc = N if ldc is None else ldc
        self.c_rows = int(self.orow0[-1] + P_out[-1] + gap)
        self.tab = _i32(np.concatenate([self.row0, self.orow0, self.t_valid]), dev)
        gen = torch.Generator().manual_seed(9000 + seed)
        self.a_rows = self.M + (K + R - 1) // R + 2
        A = torch.randn(self.a_rows * R, generator=gen)
        B = torch.randn(N * K, generator=gen) * 0.1
        self.bias = (torch.randn(N, generator=gen)).to(dev) if bias else None
        if mode is None:                                  # FFMA: plain fp32 operands
            (Ah, Al), (Bh, Bl) = (A, None), (B, None)
        else:
            (Ah, Al), (Bh, Bl) = _operands(A, mode), _operands(B, mode, weights=True)
        # the sentinel wherever no stored element reads: rows of unstored frames, slack rows
        read = torch.zeros(self.a_rows * R, dtype=torch.bool)
        for i in range(n):
            rows = -(-int(self.t_valid[i]) // fold)
            a = int(self.row0[i]) * R
            read[a:a + (rows - 1) * R + K] = True
        _poison((Ah, Al), ~read)
        self.Ah, self.Al, self.Bh, self.Bl = (None if t is None else t.to(dev)
                                              for t in (Ah, Al, Bh, Bl))
        self.cdt = torch.bfloat16 if c_bf16 else torch.float32

    def out(self):
        return _full(self.c_rows * self.ldc + 64, GUARD, self.dev, self.cdt)

    def run_var(self, stats=False):
        C = self.out()
        cs = cq = None
        if stats:
            cs = _full(self.N + 8, GUARD, self.dev, torch.float64)
            cq = _full(self.N + 8, GUARD, self.dev, torch.float64)
            cs[:self.N] = 0
            cq[:self.N] = 0
        if self.mode is None:
            args = [self.Ah, self.R, self.Bh, self.K, C, self.ldc, self.M, self.N, self.K,
                    self.bias, self.tab, self.n, self.fold]
            name = "pase_gemm_nt_var"
        else:
            args = [self.Ah, self.Al, self.a_rows, self.R, self.Bh, self.Bl, self.K, C,
                    self.ldc, self.M, self.N, self.K, self.bias, self.tab, self.n, self.fold]
            name = "pase_tc_gemm_nt_var"
        if stats:
            tail = [self.mode, self.c_bf16] if self.mode is not None else []
            _call(self.dev, name + "_stats", *(args + [cs, cq] + tail))
        else:
            _call(self.dev, name, *(args + ([self.mode, self.c_bf16]
                                             if self.mode is not None else [])))
        return C, cs, cq

    def run_uniform(self):
        """The uniform kernel as one B=1 call per utterance, into a guard-filled buffer."""
        C = self.out()
        for i in range(self.n):
            r0, P, o0, tv = int(self.row0[i]), int(self.P[i]), int(self.orow0[i]), \
                int(self.t_valid[i])
            Cv = C[o0 * self.ldc:]
            if self.mode is None:
                _call(self.dev, "pase_gemm_nt", self.Ah[r0 * self.R:], self.R, self.Bh, self.K,
                      Cv, self.ldc, P, self.N, self.K, 1.0, self.bias, P, tv, P, self.fold,
                      None, None, 0)
            else:
                lo = None if self.Al is None else self.Al[r0 * self.R:]
                _call(self.dev, "pase_tc_gemm_nt", self.Ah[r0 * self.R:], lo,
                      self.a_rows - r0, self.R, self.Bh, self.Bl, self.K, Cv, self.ldc, P,
                      self.N, self.K, 1.0, None, self.bias, P, tv, P, self.fold, None, None, 0,
                      self.mode, self.c_bf16)
        return C

    def checks(self, C, cs=None, cq=None):
        """Stored elements against float64, guards everywhere else, sums against float64
        sums of the stored values."""
        mode = 0 if self.mode is None else self.mode
        Aop = emul.core._operand(self.Ah.cpu(), None if self.Al is None else self.Al.cpu(),
                                 mode).to(self.dev).double() if self.mode is not None \
            else self.Ah.double()
        Bop = emul.core._operand(self.Bh.cpu(), None if self.Bl is None else self.Bl.cpu(),
                                 mode).to(self.dev).double() if self.mode is not None \
            else self.Bh.double()
        Bm = Bop[:self.N * self.K].view(self.N, self.K)
        out, spans = [], []
        s_sum = torch.zeros(self.N, dtype=torch.float64, device=self.dev)
        s_sq, s_abs, s_abs2 = s_sum.clone(), s_sum.clone(), s_sum.clone()
        for i in range(self.n):
            r0, P, o0, tv = int(self.row0[i]), int(self.P[i]), int(self.orow0[i]), \
                int(self.t_valid[i])
            rows = -(-tv // self.fold)
            Ar = torch.as_strided(Aop, (rows, self.K), (self.R, 1), r0 * self.R)
            ref = Ar @ Bm.t()
            mag = Ar.abs() @ Bm.abs().t()
            tol = (2 * self.K * U + 2.0 ** -20) * mag
            if self.bias is not None:
                ref = ref + self.bias.double()
                tol = tol + _ulp32(ref)
            got = torch.as_strided(C, (rows, self.N), (self.ldc, 1), o0 * self.ldc)
            if self.c_bf16:
                tol = tol + 2.0 ** -8 * ref.abs()
            mask = _stored_mask(rows, tv, self.N, self.fold, self.dev)
            out.append(("C utt %d" % i, got[mask], ref[mask], tol[mask]))
            spans += [(o0 * self.ldc + u * self.ldc, o0 * self.ldc + u * self.ldc + self.N)
                      for u in range(rows)]
            vals = torch.where(mask, got.double(), torch.zeros_like(ref))
            s_sum += vals.sum(0)
            s_sq += (vals * vals).sum(0)
            s_abs += vals.abs().sum(0)
            s_abs2 += (vals * vals).sum(0)
        # guards: every element outside the stored ones (unstored frames hold GUARD too)
        keep = torch.ones(C.numel(), dtype=torch.bool, device=self.dev)
        for i in range(self.n):
            o0, tv = int(self.orow0[i]), int(self.t_valid[i])
            rows = -(-tv // self.fold)
            mask = _stored_mask(rows, tv, self.N, self.fold, self.dev)
            torch.as_strided(keep, (rows, self.N), (self.ldc, 1), o0 * self.ldc)[mask] = False
        assert bool((C[keep] == GUARD).all()), "C: written outside the row map"
        if cs is not None:
            assert bool((cs[self.N:] == GUARD).all()) and bool((cq[self.N:] == GUARD).all())
            # the sums are those of the fp32 values; a 16-bit C stores them rounded once more
            r1, r2 = (2.0 ** -8, 2.0 ** -7) if self.c_bf16 else (0.0, 0.0)
            out += [("colsum", cs[:self.N], s_sum, (2.0 ** -16 + r1) * s_abs),
                    ("colsumsq", cq[:self.N], s_sq, (2.0 ** -16 + r2) * s_abs2)]
        return out


def _block_gemm(lengths, l, prec, mode, dev, c_bf16=0, ldc_extra=0, seed=0):
    """VarGemm of block l with the product's var_tab for these lengths (plus output gaps)."""
    plan, geoms, host, sec, sz = product_layout(lengths, prec)
    g, n = plan.geoms[l], len(lengths)
    row0, orow0, tv = _var_rows(host[sec[("gemm", l)]:], n)
    assert (orow0 == np.concatenate([[0], np.cumsum([gi[l].rows_out for gi in geoms])])[:n]).all()
    P_out = np.asarray([gi[l].rows_out for gi in geoms])
    R = g.lda
    return VarGemm(row0, tv, P_out, R, g.K, g.Nn, g.fold, mode, dev, c_bf16=c_bf16,
                   ldc=g.Nn + ldc_extra, seed=seed)


# (lengths, block, precision, mode (None: FFMA), c_bf16, extra ldc)
GEMM_CASES = {
    "ffma-sinc-fold4-edges": ("edges", 0, "fp32", None, 0, 0),
    "ffma-conv1-edges": ("edges", 1, "fp32", None, 0, 0),
    "ffma-conv2-seeded48": ("seeded48", 2, "fp32", None, 0, 0),
    "tf32-conv2-edges": ("edges", 2, "tf32", 0, 0, 0),
    "3xtf32-sinc-fold32-edges": ("edges", 0, "3xtf32", 1, 0, 0),
    "bf16-sinc-fold64-edges": ("edges", 0, "bf16", 2, 0, 0),
    "bf16-conv1-seeded48-c16": ("seeded48", 1, "bf16", 2, 1, 0),
    "3xf16-conv3-single": ("single", 3, "3xf16", 3, 0, 0),
    "3xf16-conv2-edges-c16-oddldc": ("edges", 2, "3xf16", 3, 1, 1),
}


def gemm_case(name, dev, stats):
    lists = length_lists(pasep_cfg())
    key, l, prec, mode, c16, extra = GEMM_CASES[name]
    v = _block_gemm(lists[key], l, prec, mode, dev, c_bf16=c16, ldc_extra=extra, seed=l)
    if v.fold > 1:
        assert any(int(t) % v.fold for t in v.t_valid), "no t_valid off the fold"
    C, cs, cq = v.run_var(stats)
    return v, C, cs, cq


@pytest.mark.parametrize("stats", [False, True])
@pytest.mark.parametrize("name", list(GEMM_CASES))
def test_var_gemm(name, stats):
    """Row map, guards, float64 bound, and (no statistics) bits of the uniform B=1 calls."""
    v, C, cs, cq = gemm_case(name, "cuda", stats)
    if not stats:
        assert torch.equal(C, v.run_uniform()), "packed GEMM != uniform B=1 GEMMs"
    _report("var gemm %s%s" % (name, " stats" if stats else ""), _check_all(v.checks(C, cs, cq)))


def _tail_gemm(mode, stats, c_bf16, ldc_extra=0):
    """A boundary inside the partial last round: search the rows M (N = 128) for which
    pase_tc_gemm_nt_plan leaves tail_bn != 0 on this device, and put one utterance across
    bulk_m and the last boundary inside the tail rows."""
    sms = _lib.device_info()["sms"]
    N, K, R = 128, 704, 128
    for M in range(20000, 80000, 64):
        plan = _lib.tc_gemm_nt_plan(M, N, sms)
        if plan["tail_bn"] and M - plan["bulk_m"] >= 64:
            break
    else:
        raise AssertionError("no M with a partial last round")
    bulk, used = plan["bulk_m"], M - 20
    P0 = bulk - 100
    P1 = 100 + (used - bulk) // 2
    P = [P0 - 1000, 1000, P1, used - P0 - P1]
    row0 = np.concatenate([[0], np.cumsum(P)])
    assert row0[2] < bulk < row0[3] < used and bulk < row0[3]
    tv = [p - 5 for p in P]
    tv[1] = 1
    print("tail plan M=%d N=%d on %d SMs: %s, boundaries %s" % (M, N, sms, plan,
                                                                 row0.tolist()))
    v = VarGemm(row0, tv, P, R, K, N, 1, mode, "cuda", slack=20, c_bf16=c_bf16,
                ldc=N + ldc_extra, seed=mode)
    assert v.M == M
    return v, plan


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_var_gemm_tail_round(mode):
    v, plan = _tail_gemm(mode, False, 0)
    assert plan["tail_bn"] != 0
    C, _, _ = v.run_var(False)
    assert torch.equal(C, v.run_uniform()), "packed GEMM != uniform B=1 GEMMs"
    r = _check_all(v.checks(C))
    C, cs, cq = v.run_var(True)
    r += _check_all(v.checks(C, cs, cq))
    _report("var gemm tail round mode %d" % mode, r)


@pytest.mark.parametrize("mode", [2, 3])
def test_var_gemm_bf16_out_odd_ldc(mode):
    """16-bit C with an odd ldc: the scalar store path, across the partial last round too."""
    v, plan = _tail_gemm(mode, False, 1, ldc_extra=1)
    assert v.ldc % 2 == 1
    C, _, _ = v.run_var(False)
    assert torch.equal(C, v.run_uniform()), "packed GEMM != uniform B=1 GEMMs"
    _report("var gemm bf16 out ldc %d mode %d" % (v.ldc, mode), _check_all(v.checks(C)))


# ================================ waveform pad and fold ================================
class Wave(object):
    """Utterances of `lengths` packed in x with gaps; dst regions with gaps (the product's
    wave section gives the offsets, plus `gap` elements between regions)."""

    def __init__(self, lengths, padL, padR, dev, gap=5, seed=0):
        self.lengths, self.padL, self.padR, self.dev = list(lengths), padL, padR, dev
        n = len(lengths)
        gen = torch.Generator().manual_seed(8000 + seed)
        self.x_off = np.concatenate([[0], np.cumsum(np.asarray(lengths) + gap)])[:n]
        self.d_off = np.concatenate([[0], np.cumsum(np.asarray(lengths) + padL + padR + gap)])[:n]
        self.nx = int(self.x_off[-1] + lengths[-1] + gap)
        self.nd = int(self.d_off[-1] + lengths[-1] + padL + padR + gap)
        x = torch.full((self.nx,), SENT)
        for o, T in zip(self.x_off, lengths):
            x[o:o + T] = torch.randn(T, generator=gen)
        self.x = x.to(dev)
        self.tab = _i32(np.stack([self.x_off, lengths, self.d_off], 1), dev)
        self.max_T = max(lengths)
        d = torch.full((self.nd,), SENT)
        for o, T in zip(self.d_off, lengths):
            d[o:o + T + padL + padR] = torch.randn(T + padL + padR, generator=gen)
        self.dpad = d.to(dev)

    def ref_pad(self, i):
        o, T = int(self.x_off[i]), self.lengths[i]
        idx = emul.core._reflect(torch.arange(T + self.padL + self.padR) - self.padL, T)
        return self.x[o:o + T].double()[idx.to(self.dev)]

    def ref_fold(self, i, fold_l=1, fold_r=1):
        """float64 fold of utterance i's pad gradient and the magnitudes of its terms."""
        o, T, pL, pR = int(self.d_off[i]), self.lengths[i], self.padL, self.padR
        d = self.dpad[o:o + T + pL + pR].double()
        idx = emul.core._reflect(torch.arange(T + pL + pR) - pL, T).to(self.dev)
        keep = torch.ones(T + pL + pR, dtype=torch.bool, device=self.dev)
        if not fold_l:
            keep[:pL] = False
        if not fold_r:
            keep[T + pL:] = False
        ref = torch.zeros(T, dtype=torch.float64, device=self.dev)
        mag = torch.zeros_like(ref)
        ref.index_add_(0, idx[keep], d[keep])
        mag.index_add_(0, idx[keep], d[keep].abs())
        return ref, mag


def pad_checks(w, fmt):
    dt = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}[fmt]
    g = GUARD if fmt != 2 else F16_SENT
    dst = _full(w.nd, g, w.dev, dt)
    lo = _full(w.nd, g, w.dev, dt) if fmt == 2 else None
    _call(w.dev, "pase_reflect_pad_wave_var", w.x, w.tab, len(w.lengths), w.max_T, dst, lo, fmt,
          w.padL, w.padR)
    spans, out = [], []
    for i, T in enumerate(w.lengths):
        o, n = int(w.d_off[i]), T + w.padL + w.padR
        spans.append((o, o + n))
        ref = w.ref_pad(i).float()
        if fmt == 0:
            assert torch.equal(dst[o:o + n], ref), "fp32 pad not exact (utt %d)" % i
        elif fmt == 1:
            assert torch.equal(dst[o:o + n], ref.to(torch.bfloat16)), "bf16 pad (utt %d)" % i
        else:
            hi = ref.to(torch.float16)
            assert torch.equal(dst[o:o + n], hi), "fp16 hi (utt %d)" % i
            assert torch.equal(lo[o:o + n], ((ref - hi.float()) * 2048.0).to(torch.float16)), \
                "fp16 lo (utt %d)" % i
        val = dst[o:o + n].double()
        if fmt == 2:
            val = val + lo[o:o + n].double() / 2048.0
        rel = {0: 0.0, 1: 2.0 ** -8, 2: 2.0 ** -22}[fmt]
        sub = 2.0 ** -35 if fmt == 2 else 0.0          # half the fp16 subnormal step of lo
        out.append(("pad %d fmt %d" % (i, fmt), val, ref.double(),
                    rel * ref.double().abs() + sub))
    _unchanged("pad dst", dst, spans, g)
    if lo is not None:
        _unchanged("pad dst_lo", lo, spans, g)
    return dst, lo, out


def fold_checks(w):
    dx = _full(w.nx, GUARD, w.dev)
    _call(w.dev, "pase_reflect_fold_wave_var", w.dpad, w.tab, len(w.lengths), w.max_T, dx,
          w.padL, w.padR)
    out, spans = [], []
    for i, T in enumerate(w.lengths):
        o = int(w.x_off[i])
        ref, mag = w.ref_fold(i)
        out.append(("fold %d" % i, dx[o:o + T], ref, 2 * U * mag))
        spans.append((o, o + T))
        # adjoint: <pad(x), d> == <x, fold_kernel(d)> in float64, within the fold's bound
        od = int(w.d_off[i])
        d = w.dpad[od:od + T + w.padL + w.padR].double()
        xv = w.x[o:o + T].double()
        lhs = float((w.ref_pad(i) * d).sum())
        rhs = float((xv * dx[o:o + T].double()).sum())
        slack = float((xv.abs() * 2 * U * mag).sum()) + 1e-12 * float((xv.abs() * mag).sum())
        assert abs(lhs - rhs) <= slack, "pad and fold are not adjoint (utt %d)" % i
    _unchanged("fold dx", dx, spans, GUARD)
    return dx, out


def fold_acc_checks(dev, seed=0):
    """Overlapping windows of one recording folded into dx in order, each of the four
    (fold_l, fold_r) cases once; dx accumulates."""
    gen = torch.Generator().manual_seed(8100 + seed)
    L, pL, pR, base = 3000, 125, 125, 40
    wins = [(0, 900, 1, 0), (700, 1000, 0, 0), (1600, 1400, 0, 1), (1000, 1100, 1, 1)]
    x0s = [(base + a, T, fl, fr) for a, T, fl, fr in wins]
    dx = _full(base + L + 40, GUARD, dev)
    dx[base:base + L] = torch.randn(L, generator=gen).to(dev)
    ref = dx[base:base + L].double().clone()
    mag = ref.abs()
    for x0, T, fl, fr in x0s:
        d = torch.randn(T + pL + pR, generator=gen).to(dev)
        _call(dev, "pase_reflect_fold_wave_acc", d, dx, x0, T, pL, pR, fl, fr)
        idx = emul.core._reflect(torch.arange(T + pL + pR) - pL, T).to(dev)
        keep = torch.ones(T + pL + pR, dtype=torch.bool, device=dev)
        if not fl:
            keep[:pL] = False
        if not fr:
            keep[T + pL:] = False
        add = torch.zeros(T, dtype=torch.float64, device=dev)
        am = torch.zeros_like(add)
        add.index_add_(0, idx[keep], d.double()[keep])
        am.index_add_(0, idx[keep], d.double().abs()[keep])
        ref[x0 - base:x0 - base + T] += add
        mag[x0 - base:x0 - base + T] += am + ref[x0 - base:x0 - base + T].abs()
    _unchanged("fold_acc dx", dx, [(base, base + L)], GUARD)
    return [("fold_acc", dx[base:base + L], ref, 2 * U * mag)]


@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("key", ["edges", "seeded48", "single"])
def test_reflect_pad_and_fold_var(key, fmt):
    lengths = length_lists(pasep_cfg())[key]
    plan, geoms, host, sec, sz = product_layout(lengths)
    g = plan.geoms[0]
    wave = host[sec["wave"]:sec["wave"] + 3 * len(lengths)].reshape(-1, 3)
    assert (wave[:, 1] == lengths).all() and (wave[:, 2] % g.lda == 0).all()
    w = Wave(lengths, g.padL, g.padR, "cuda", seed=fmt)
    dst, lo, r = pad_checks(w, fmt)
    for i, T in enumerate(lengths):            # bits of the uniform B=1 pad
        o, n = int(w.d_off[i]), T + g.padL + g.padR
        d1 = _full(n, 0.0, "cuda", dst.dtype)
        l1 = _full(n, 0.0, "cuda", dst.dtype) if lo is not None else None
        _call("cuda", "pase_reflect_pad_wave", w.x[int(w.x_off[i]):], d1, l1, fmt, 1, T, g.padL,
              g.padR, n)
        assert torch.equal(d1, dst[o:o + n]) and (lo is None or torch.equal(l1, lo[o:o + n]))
    dx, rf = fold_checks(w)
    for i, T in enumerate(lengths):            # bits of the uniform B=1 fold
        d1 = _full(T, 0.0, "cuda")
        _call("cuda", "pase_reflect_fold_wave", w.dpad[int(w.d_off[i]):], T + g.padL + g.padR,
              d1, 1, T, g.padL, g.padR)
        assert torch.equal(d1, dx[int(w.x_off[i]):int(w.x_off[i]) + T])
    _report("pad/fold %s fmt %d" % (key, fmt), _check_all(r + rf))


def test_reflect_fold_wave_acc():
    _report("fold_acc", _check_all(fold_acc_checks("cuda")))


# ================================ BatchNorm / PReLU ================================
# Storage of each encoder precision (test_bn_prelu_gpu.PRECS): y bf16, gradient source bf16,
# backward dst format; the forward writes dst in the same format.
BN_PRECS = {"fp32": (0, 0, 0), "bf16": (1, 1, 1), "bf16-a32": (1, 0, 1), "3xf16": (0, 0, 2)}
FMT_DT = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}


def _bn_params(C, gen, dev):
    rn = lambda s=1.0: (torch.randn(C, generator=gen) * s).to(dev)
    return dict(mean=rn(0.1), invstd=rn().abs() + 0.5, gamma=rn(), scale=rn(), shift=rn(0.5),
                alpha=rn(0.3))


def _away_from_kink(v, p, dt):
    """v in storage type dt, every value at least 1e-3 from its channel's PReLU kink."""
    kink = (-p["shift"].double() / p["scale"].double()).cpu()
    for step in (0.05, 0.2, 1.0, None):
        v = v.to(dt).float()
        near = (v.double() - kink).abs() < 1e-3
        if not bool(near.any()):
            return v.to(dt)
        assert step is not None, "could not move y away from the PReLU kink"
        away = torch.where(v.double() >= kink, 1.0, -1.0)
        v = torch.where(near, (kink + away * step).float(), v)


def pool_rule(Ts, Tq):
    """The product's dense-skip pooling of a block (DESIGN.md section 11): utterance i pools
    pool_T = T'_i windows of pool_d = max(T_i // T'_i, 1) frames."""
    Tq = np.asarray(Tq, np.int64)
    return Tq, np.maximum(np.asarray(Ts, np.int64) // Tq, 1)


def product_bn_rows(key, l, prec="fp32"):
    """(T, pool_T, pool_d, C) of block l for these lengths, from packed_grad_layout's backward
    section: the rows the product uploads."""
    lengths = length_lists(pasep_cfg())[key]
    plan, geoms, host, sec, sz = product_layout(lengths, prec.split("-")[0])
    n = len(lengths)
    r = host[sec[("bwd", l)]:sec[("bwd", l)] + 9 * n].reshape(n, 9)
    fw = host[sec[("bn", l)]:sec[("bn", l)] + 6 * n].reshape(n, 6)
    assert (fw[:, 4:6] == r[:, 5:7]).all() and (fw[:, 0] == r[:, 0]).all()
    assert (r[:, 6] == sz["Tq"]).all()
    assert (r[:, 5] == pool_rule(r[:, 0], r[:, 6])[1]).all()
    return r[:, 0].tolist(), r[:, 6], r[:, 5], plan.geoms[l].Cout


class BnVar(object):
    """Packed BatchNorm/PReLU operands of one block: y rows of every utterance (with gaps), the
    gradient source srcA (one row per frame, a_row_stride C, no pad), the pooled dense-skip
    gradient of each utterance's own pool_T rows, and the backward table {T, y_off, a_off,
    b_off, pool_off, pool_d, pool_T, d_off, d_span} with d_span - T zero frames after each
    utterance and `lead` before the first.  pool: (pool_T, pool_d) per utterance (pool_rule)."""

    def __init__(self, Ts, C, dev, pool, prec="fp32", lead=3, tail=4, gap=2, order=None,
                 seed=0):
        self.Ts, self.C, self.dev, self.lead = list(Ts), C, dev, lead
        self.ybf, self.abf, self.fmt = BN_PRECS[prec]
        ydt = torch.bfloat16 if self.ybf else torch.float32
        adt = torch.bfloat16 if self.abf else torch.float32
        gen = torch.Generator().manual_seed(7700 + seed)
        self.p = _bn_params(C, gen, dev)
        n = len(Ts)
        self.n = n
        pT, pd = (np.asarray(v, np.int64) for v in pool)
        assert (pT * pd <= np.asarray(Ts)).all()
        y_off = np.concatenate([[0], np.cumsum((np.asarray(Ts) + gap) * C)])[:n]
        self.ny = int(y_off[-1] + (Ts[-1] + gap) * C)
        y = torch.full((self.ny,), SENT, dtype=ydt)
        A = torch.full((self.ny,), SENT, dtype=adt)
        pc = {k: v.cpu() for k, v in self.p.items()}
        for o, T in zip(y_off, Ts):
            y[o:o + T * C] = _away_from_kink(torch.randn(T, C, generator=gen) * 1.5, pc,
                                             ydt).reshape(-1)
            A[o:o + T * C] = torch.randn(T * C, generator=gen).to(adt)
        self.y, self.A = y.to(dev), A.to(dev)
        pool_off = np.concatenate([[0], np.cumsum((pT + 1) * C)])[:n]
        pool = torch.full((int(pool_off[-1] + (pT[-1] + 1) * C),), SENT)
        for o, t in zip(pool_off, pT):
            pool[o:o + t * C] = torch.randn(int(t) * C, generator=gen)
        self.pool = pool.to(dev)
        order = list(range(n)) if order is None else order
        span = np.asarray(Ts) + tail
        d_off = np.zeros(n, np.int64)
        pos = lead
        for i in order:
            d_off[i] = pos * C
            pos += int(span[i])
        self.nd = (pos + 2) * C
        self.d_off, self.span = d_off, span
        self.rows = np.stack([Ts, y_off, y_off, np.zeros(n), pool_off, pd, pT, d_off, span],
                             1).astype(np.int64)
        self.tab = _i32(self.rows[order], dev)
        self.order = order
        self.max_T, self.max_span = max(Ts), int(span.max())

    def g_du(self, i):
        """float64 gradient sources g, the fp32 affine u, du and its magnitude bound, xhat."""
        T, yo, ao, _, po, pd, pT, _, _ = (int(v) for v in self.rows[i])
        C, p = self.C, self.p
        a = self.A[ao:ao + T * C].view(T, C).double()
        g, gabs = a.clone(), a.abs()
        pool = self.pool[po:po + pT * C].view(pT, C).double()
        g[:pT * pd] += (pool / pd).repeat_interleave(pd, 0)
        gabs[:pT * pd] += (pool.abs() / pd).repeat_interleave(pd, 0)
        y = self.y[yo:yo + T * C].view(T, C).float()
        # the kernel's fmaf(y, scale, shift): the exact float64 value rounded once to fp32
        u = (y.double() * p["scale"].double() + p["shift"].double()).float()
        al = p["alpha"].double()
        du = torch.where(u > 0, g, al * g)
        dabs = torch.where(u > 0, gabs, al.abs() * gabs)
        xh = (y.double() - p["mean"].double()) * p["invstd"].double()
        return g, u.double(), du, dabs, xh

    def reduce(self):
        C = self.C
        S1, S2, da = (_full(C + 8, GUARD, self.dev, torch.float64) for _ in range(3))
        for s in (S1, S2, da):
            s[:C] = 0
        amax = _full(4, GUARD, self.dev)
        amax[:2] = 0
        p = self.p
        _call(self.dev, "pase_bn_prelu_bwd_reduce_var", self.y, self.ybf, self.tab, self.n,
              self.max_T, C, p["mean"], p["invstd"], p["scale"], p["shift"], p["alpha"], self.A,
              self.abf, C, 0, 0, None, C, 0, self.pool, C, S1, S2, da, amax)
        return S1, S2, da, amax

    def apply(self, train=None, amax=None, fmt=None):
        C, p = self.C, self.p
        fmt = self.fmt if fmt is None else fmt
        g = F16_SENT if fmt == 2 else SENT
        dst = _full(self.nd, g, self.dev, FMT_DT[fmt])
        lo = _full(self.nd, g, self.dev, FMT_DT[fmt]) if fmt == 2 else None
        db = _full(C + 8, GUARD, self.dev, torch.float64)
        db[:C] = 0
        so = _full(4, GUARD, self.dev) if fmt == 2 else None
        common = [p["scale"], p["shift"], p["alpha"]]
        tail = [self.A, self.abf, C, 0, 0, None, C, 0, self.pool, C, dst, lo, fmt, self.lead, db,
                amax, so]
        if train is None:
            _call(self.dev, "pase_bn_prelu_bwd_apply_src_var", self.y, self.ybf, self.tab, self.n,
                  self.max_span, C, p["invstd"], p["gamma"], *common, *tail)
        else:
            S1, S2, count = train
            _call(self.dev, "pase_bn_prelu_bwd_apply_src_var_train", self.y, self.ybf, self.tab,
                  self.n, self.max_span, C, p["mean"], p["invstd"], p["gamma"], *common, S1, S2,
                  count, *tail)
        return dst, lo, db, so


def bn_reduce_checks(b):
    S1, S2, da, amax = b.reduce()
    C = b.C
    s1, s2, sa = (torch.zeros(C, dtype=torch.float64, device=b.dev) for _ in range(3))
    m1, m2, ma = (torch.zeros(C, dtype=torch.float64, device=b.dev) for _ in range(3))
    dmax, xmax = 0.0, 0.0
    for i in range(b.n):
        g, u, du, dabs, xh = b.g_du(i)
        s1 += du.sum(0)
        m1 += dabs.sum(0)
        s2 += (du * xh).sum(0)
        m2 += (dabs * xh.abs()).sum(0)
        neg = u <= 0
        sa += torch.where(neg, u * g, torch.zeros_like(g)).sum(0)
        ma += torch.where(neg, (u * g).abs(), torch.zeros_like(g)).sum(0)
        dmax, xmax = max(dmax, float(du.abs().max())), max(xmax, float(xh.abs().max()))
    for s in (S1, S2, da):
        assert bool((s[C:] == GUARD).all()), "sums: guard written"
    assert bool((amax[2:] == GUARD).all()), "amax: guard written"
    count = float(sum(b.Ts))
    one = lambda v: torch.tensor([v], dtype=torch.float64, device=b.dev)
    return (S1, S2, count), amax, [
        ("S1", S1[:C], s1, 2.0 ** -16 * m1), ("S2", S2[:C], s2, 2.0 ** -16 * m2),
        ("dalpha", da[:C], sa, 2.0 ** -16 * ma),
        ("amax du", amax[:1], one(dmax), one(2.0 ** -20 * dmax)),
        ("amax xhat", amax[1:2], one(xmax), one(2.0 ** -20 * xmax))]


def bn_apply_checks(b, dst, db, train=None, lo=None, so=None):
    """dy of every utterance within the bound (bf16: plus one rounding; fp16 pair: hi + lo/2^11
    unscaled by scale_out), zero frames [T, d_span) and the lead zero, everything else
    untouched; dbias within 2^-16."""
    C, p = b.C, b.p
    gi = (p["gamma"].double() * p["invstd"].double())
    out, spans = [], [(0, b.lead * C)]
    dbr = torch.zeros(C, dtype=torch.float64, device=b.dev)
    dbm = torch.zeros_like(dbr)
    assert int(b.d_off[b.order[0]]) == b.lead * C
    for i in range(b.n):
        T, d0, span = b.Ts[i], int(b.d_off[i]), int(b.span[i])
        g, u, du, dabs, xh = b.g_du(i)
        if train is None:
            ref = gi * du
            tol = 2.0 ** -20 * gi.abs() * dabs
        else:
            S1, S2, count = train
            m1, m2 = S1[:C] / count, S2[:C] / count
            ref = gi * (du - m1 - xh * m2)
            tol = 2.0 ** -20 * gi.abs() * (dabs + m1.abs() + xh.abs() * m2.abs())
        got = dst[d0:d0 + T * C].view(T, C).double()
        if dst.dtype == torch.bfloat16:
            tol = tol + 2.0 ** -8 * ref.abs()
        elif dst.dtype == torch.float16:
            got = (got + lo[d0:d0 + T * C].view(T, C).double() / 2048.0) * float(so[0])
            tol = tol + 2.0 ** -21 * ref.abs() + 2.0 ** -35 * float(so[0])
        out.append(("dy %d" % i, got, ref, tol))
        dbr += ref.sum(0)
        dbm += ref.abs().sum(0)
        for buf in (dst,) if lo is None else (dst, lo):
            assert bool((buf[d0 + T * C:d0 + span * C] == 0).all()), \
                "zero frames [T, d_span) of utterance %d not written" % i
        spans.append((d0, d0 + span * C))
    for buf in (dst,) if lo is None else (dst, lo):
        assert bool((buf[:b.lead * C] == 0).all()), "lead frames not written zero"
        _unchanged("dst", buf, spans, SENT if buf.dtype != torch.float16 else F16_SENT)
    assert bool((db[C:] == GUARD).all())
    # dbias sums the values before the 16-bit rounding of dst
    out.append(("dbias", db[:C], dbr, 2.0 ** -16 * dbm + 2.0 ** -20 * dbm))
    return out


def bn_fwd_checks(b, sep=1, pool=True, padL=0, padR=0):
    """pase_bn_prelu_pad_fwd_var in b's precision (y bf16 or fp32; dst fp32, bf16 or the fp16
    pair): dst rows [sep row | padded frames] per utterance with a gap row, each utterance's
    pool_T pooled rows (pool_d frames each, the rest of its frames unpooled) into pool columns
    [0, C) of rows of pitch C + 8."""
    C, p, n, fmt = b.C, b.p, b.n, b.fmt
    assert min(b.Ts) > max(padL, padR), "a reflect pad needs T > pad"
    Tp = [T + padL + padR for T in b.Ts]
    d_off = np.concatenate([[1], np.cumsum(np.asarray(Tp) + 2) + 1])[:n] * C
    nd = int(d_off[-1] + (Tp[-1] + 2) * C)
    prs = C + 8
    pT, pd = b.rows[:, 6], b.rows[:, 5]
    pool_off = np.concatenate([[0], np.cumsum((pT + 1) * prs)])[:n]
    y_off = b.rows[:, 1]
    tab = _i32(np.stack([b.Ts, y_off, d_off, pool_off, pd, pT], 1), b.dev)
    g = F16_SENT if fmt == 2 else GUARD
    dst = _full(nd, g, b.dev, FMT_DT[fmt])
    lo = _full(nd, g, b.dev, FMT_DT[fmt]) if fmt == 2 else None
    pl = _full(int(pool_off[-1] + (pT[-1] + 1) * prs), GUARD, b.dev) if pool else None
    if pool:
        for o, t in zip(pool_off, pT):
            torch.as_strided(pl, (int(t), C), (prs, 1), int(o)).zero_()
    _call(b.dev, "pase_bn_prelu_pad_fwd_var", b.y, b.ybf, tab, n, b.max_T, C, p["scale"],
          p["shift"], p["alpha"], dst, lo, fmt, C, padL, padR, pl, prs, sep)
    out, spans, pspans = [], [], []
    for i, T in enumerate(b.Ts):
        yo, d0 = int(y_off[i]), int(d_off[i])
        y = b.y[yo:yo + T * C].view(T, C).float()
        gate = torch.where(y * p["scale"] + p["shift"] > 0, 1.0, p["alpha"].double())
        a = gate * (y.double() * p["scale"].double() + p["shift"].double())
        # the fp32 affine rounds relative to its terms, then the gate's product once more
        am = gate.abs() * 2 * U * ((y.double() * p["scale"].double()).abs()
                                   + p["shift"].double().abs())
        idx = emul.core._reflect(torch.arange(Tp[i]) - padL, T).to(b.dev)
        ref = a[idx]
        got = dst[d0:d0 + Tp[i] * C].view(Tp[i], C).double()
        tol = am[idx] + 2 * _ulp32(ref)
        if fmt == 1:
            tol = tol + 2.0 ** -8 * ref.abs()
        elif fmt == 2:
            got = got + lo[d0:d0 + Tp[i] * C].view(Tp[i], C).double() / 2048.0
            tol = tol + 2.0 ** -22 * ref.abs() + 2.0 ** -35
        out.append(("fwd %d" % i, got, ref, tol))
        spans.append((d0, d0 + Tp[i] * C))
        if sep:
            assert bool((dst[d0 - C:d0] == 0).all()), "sep row of utterance %d" % i
            spans.append((d0 - C, d0))
        if pool:
            t, d = int(pT[i]), int(pd[i])
            pv = torch.as_strided(pl, (t, C), (prs, 1), int(pool_off[i]))
            # the pooled value is the stored activation (what the next layer reads)
            # the pooled value is the stored activation (what the next layer reads); the fp16
            # pair's lo may be subnormal
            seen = got[padL:padL + t * d].view(t, d, C)
            out.append(("pool %d" % i, pv, seen.mean(1), (d + 4) * U * seen.abs().mean(1)
                        + (2.0 ** -35 if fmt == 2 else 0.0)))
            pspans += [(int(pool_off[i]) + j * prs, int(pool_off[i]) + j * prs + C)
                       for j in range(t)]
    for buf in (dst,) if lo is None else (dst, lo):
        _unchanged("fwd dst", buf, spans, g)
    if pool:
        _unchanged("pool columns", pl, pspans, GUARD)
    return tab, dst, lo, pl, out


# (lengths, block) of the product's tables: block 1 (C 64) of the edge lengths, T'_i from 3 to
# 513, every pool_T * pool_d < T; block 6 (C 512) of 48 seeded lengths
BN_CASES = {"edges-block1": ("edges", 1), "seeded48-block6": ("seeded48", 6),
            "single-block3": ("single", 3)}


def _bn_case(case, prec, seed, **kw):
    key, l = BN_CASES[case]
    Ts, pT, pd, C = product_bn_rows(key, l, prec)
    return BnVar(Ts, C, "cuda", (pT, pd), prec=prec, seed=seed, **kw)


@pytest.mark.parametrize("prec", list(BN_PRECS))
@pytest.mark.parametrize("case", list(BN_CASES))
def test_bn_prelu_pad_fwd_var(case, prec):
    b = _bn_case(case, prec, 1)
    assert any(int(r[5]) * int(r[6]) < int(r[0]) for r in b.rows), "no unpooled frames"
    assert b.n == 1 or len({int(r[6]) for r in b.rows}) > 1, "one pool_T for every row"
    tab, dst, lo, pl, r = bn_fwd_checks(b, sep=1, pool=True)
    # bits of the uniform B=1 forward on the same offsets
    C, p = b.C, b.p
    for T, yo, do, po, pd, pT in tab.view(-1, 6).tolist():
        d1 = _full(T * C, 0.0, "cuda", dst.dtype)
        l1 = _full(T * C, 0.0, "cuda", dst.dtype) if lo is not None else None
        p1 = torch.zeros(pT * (C + 8), device="cuda")
        _call("cuda", "pase_bn_prelu_pad_fwd", b.y[yo:], b.ybf, 0, 1, T, C, p["scale"],
              p["shift"], p["alpha"], d1, l1, b.fmt, 0, C, 0, 0, p1, 0, C + 8, pd, pT)
        assert torch.equal(d1, dst[do:do + T * C])
        assert lo is None or torch.equal(l1, lo[do:do + T * C])
        assert torch.equal(torch.as_strided(p1, (pT, C), (C + 8, 1)),
                           torch.as_strided(pl, (pT, C), (C + 8, 1), po))
    # padded rows with a reflect halo, no pool (the conv blocks' operand)
    r2 = bn_fwd_checks(b, sep=0, pool=False, padL=5, padR=5)[4]
    _report("bn fwd var %s %s" % (case, prec), _check_all(r + r2))


@pytest.mark.parametrize("prec", list(BN_PRECS))
@pytest.mark.parametrize("case", list(BN_CASES))
def test_bn_prelu_bwd_var_eval(case, prec):
    """Eval mode: sums against float64, dy against float64 and bit for bit against
    pase_bn_prelu_bwd_apply_src at N = 1 on the same offsets with the pack-wide amax; zero
    frames written on every call, also where the previous call (another utterance order) left
    data; the fp16-pair scale_out derived from the pack-wide amax."""
    b = _bn_case(case, prec, 2)
    _, amax, r = bn_reduce_checks(b)
    r = _check_all(r)
    dst, lo, db, so = b.apply(amax=amax)
    r += _check_all(bn_apply_checks(b, dst, db, lo=lo, so=so))
    C, p = b.C, b.p
    zero = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    so1 = torch.zeros(2, device="cuda") if so is not None else None
    for T, yo, ao, _, po, pd, pT, do, span in b.rows.tolist():
        d1 = _full(T * C, 0.0, "cuda", dst.dtype)
        l1 = _full(T * C, 0.0, "cuda", dst.dtype) if lo is not None else None
        _call("cuda", "pase_bn_prelu_bwd_apply_src", b.y[yo:], b.ybf, 0, 1, T, C, p["mean"],
              p["invstd"], p["gamma"], p["scale"], p["shift"], p["alpha"], zero[:C], zero[C:],
              1.0, b.A[ao:], b.abf, 0, C, 0, 0, None, 0, C, 0, b.pool[po:], 0, C, pd, pT, d1, l1,
              b.fmt, 0, None, amax if so is not None else None, so1)
        assert torch.equal(d1, dst[do:do + T * C]), "packed apply != B=1 apply_src"
        assert lo is None or torch.equal(l1, lo[do:do + T * C])
    if so is not None:
        assert torch.equal(so[:2], so1) and bool((so[2:] == GUARD).all()), (so, so1)
        s = float(so[1])
        assert s == 2.0 ** round(np.log2(s)) and float(so[0]) * s == 1.0
    # a second call with the utterances in reverse order, into the same (now dirty) buffer
    key, l = BN_CASES[case]
    Ts, pT, pd, _ = product_bn_rows(key, l, prec)
    b2 = BnVar(Ts, C, "cuda", (pT, pd), prec=prec, seed=2, order=list(range(b.n))[::-1])
    assert b2.nd == b.nd
    dirty, dlo = dst.clone(), None if lo is None else lo.clone()
    _call("cuda", "pase_bn_prelu_bwd_apply_src_var", b2.y, b2.ybf, b2.tab, b2.n, b2.max_span, C,
          p["invstd"], p["gamma"], p["scale"], p["shift"], p["alpha"], b2.A, b2.abf, C, 0, 0,
          None, C, 0, b2.pool, C, dirty, dlo, b2.fmt, b2.lead, None,
          amax if so is not None else None, so1)
    for buf in (dirty,) if dlo is None else (dirty, dlo):
        for i in range(b2.n):
            T, d0, span = Ts[i], int(b2.d_off[i]), int(b2.span[i])
            assert bool((buf[d0 + T * C:d0 + span * C] == 0).all()), "stale data in zero frames"
        assert bool((buf[:b2.lead * C] == 0).all())
    _report("bn bwd var eval %s %s" % (case, prec), r)


@pytest.mark.parametrize("prec", list(BN_PRECS))
@pytest.mark.parametrize("case", list(BN_CASES))
def test_bn_prelu_bwd_var_train(case, prec):
    """Train mode: dy = gamma invstd (du - S1/count - xhat S2/count) over the whole pack."""
    b = _bn_case(case, prec, 3)
    train, amax, r = bn_reduce_checks(b)
    r = _check_all(r)
    dst, lo, db, so = b.apply(train=train, amax=amax)
    r += _check_all(bn_apply_checks(b, dst, db, train, lo=lo, so=so))
    _report("bn bwd var train %s %s" % (case, prec), r)


# ================================ QRNN ================================
QRNN_TS = (1, 16, 17, 300, 512, 513, 2000)


def _expected_width(T):
    nseg = -(-T // 16)
    return 16 if nseg <= 16 else 24 if nseg <= 24 else 32 if nseg <= 32 else 0


class QrnnVar(object):
    """Utterances of Ts packed with `gap` sentinel rows between them; each one's operands are
    those of a B=1 Qrnn (test_qrnn_sinc_out_gpu), which runs the uniform kernels."""

    def __init__(self, Ts, H, dev, gap=2, seed=0):
        self.Ts, self.H, self.dev = list(Ts), H, dev
        self.ld = H + 8
        self.qs = [Qrnn(1, T, H, ld=self.ld, dev=dev, seed=seed + i) for i, T in enumerate(Ts)]
        n = len(Ts)
        self.row0 = np.concatenate([[0], np.cumsum(np.asarray(Ts) + gap)])[:n]
        self.drow0 = np.concatenate([[0], np.cumsum(np.asarray(Ts) + 1 + gap)])[:n]
        R = int(self.row0[-1] + Ts[-1] + gap)
        Rd = int(self.drow0[-1] + Ts[-1] + 1 + gap)
        self.Y = _full(R * 3 * H + 64, SENT, dev)
        self.dh = _full((R + 2) * self.ld, SENT, dev)
        for q, r0, T in zip(self.qs, self.row0, Ts):
            self.Y[r0 * 3 * H:(r0 + T) * 3 * H] = q.Y[:T * 3 * H]
            torch.as_strided(self.dh, (T, H), (self.ld, 1), int(r0) * self.ld).copy_(
                q.hview(q.dh)[0])
        self.h = _full((R + 16) * self.ld, GUARD, dev)
        self.Cst = _full((R + 16) * H, GUARD, dev)
        self.dY = _full(Rd * 3 * H + 64, GUARD, dev)
        self.fwd_tab = _i32(np.stack([self.row0, Ts], 1), dev)
        self.bwd_tab = _i32(np.stack([self.row0, Ts, self.drow0], 1), dev)

    def run(self):
        n, H = len(self.Ts), self.H
        _call(self.dev, "pase_qrnn_scan_fwd_var", self.Y, self.h, self.ld, self.Cst,
              self.fwd_tab, n, H)
        _call(self.dev, "pase_qrnn_scan_bwd_var", self.Y, self.Cst, self.dh, self.ld, self.dY,
              self.bwd_tab, n, H)

    def checks(self, uniform_bits):
        """Each utterance's results copied into its Qrnn (after comparing with the uniform
        kernels' bits when asked) and checked there against float64; guards and the zero
        row drow0 + T."""
        H, ld, out = self.H, self.ld, []
        hs, cs, ds = [], [], []
        for q, r0, dr0, T in zip(self.qs, self.row0, self.drow0, self.Ts):
            r0, dr0 = int(r0), int(dr0)
            h = torch.as_strided(self.h, (1, T, H), (T * ld, ld, 1), r0 * ld)
            C = self.Cst[r0 * H:(r0 + T) * H]
            dY = self.dY[dr0 * 3 * H:(dr0 + T) * 3 * H]
            if uniform_bits:
                q.fwd()
                q.bwd()
                assert torch.equal(q.hview(q.h), h), "h != B=1 scan (T=%d)" % T
                assert torch.equal(q.Cst[:T * H], C), "Cst != B=1 scan (T=%d)" % T
                assert torch.equal(q.dY[:T * 3 * H], dY), "dY != B=1 scan (T=%d)" % T
            q.hview(q.h).copy_(h)
            q.Cst[:T * H] = C
            q.dY[:T * 3 * H] = dY
            assert bool((self.dY[(dr0 + T) * 3 * H:(dr0 + T + 1) * 3 * H] == 0).all()), \
                "row drow0 + T of dY not zero (T=%d)" % T
            out += [("T=%d %s" % (T, w), g, r, t) for (w, g, r, t) in
                    qrnn_fwd_checks(q) + qrnn_bwd_checks(q)]
            hs += [(r0 * ld + t * ld, r0 * ld + t * ld + H) for t in range(T)]
            cs.append((r0 * H, (r0 + T) * H))
            ds.append((dr0 * 3 * H, (dr0 + T + 1) * 3 * H))
        _unchanged("h", self.h, hs, GUARD)
        _unchanged("Cst", self.Cst, cs, GUARD)
        _unchanged("dY", self.dY, ds, GUARD)
        return out


def test_qrnn_scan_var_mixed_lengths():
    """One launch pair holding T' = 1, 16, 17, 300, 512, 513 and 2000: every algorithm."""
    for T in QRNN_TS:
        w = _lib.qrnn_scan_plan(T)
        assert w == _expected_width(T), (T, w)
        print("qrnn plan T'=%d: %s" % (T, "segments/block %d" % w if w else "sequential"))
    assert {_expected_width(T) for T in QRNN_TS} == {0, 16, 24, 32}
    v = QrnnVar(QRNN_TS, 100, "cuda", seed=40)
    v.run()
    _report("qrnn var mixed", _check_all(v.checks(True)))


def test_qrnn_scan_var_pasep_width():
    """H = 512 (PASE+) at the pitch of the concatenated operand, utterance order shuffled."""
    v = QrnnVar((513, 3, 512, 48, 1), 512, "cuda", seed=50)
    v.run()
    _report("qrnn var H=512", _check_all(v.checks(True)))


def qrnn_carry_checks(dev, H=64, seed=60):
    """Two recordings scanned window by window in three launches (a slot at most once per
    launch): A (1100 frames, slot 1) in windows [0,400) [400,800) [800,1100), B (700 frames,
    slot 3) in [0,350) [350,700).  State rows 0 and 2 are never touched; first != 0 ignores
    the slot's old state (the sentinel).  Then the backward in reverse window order with the
    logged entering states, crops c0 > 0 inside each window and a zero dstate to start."""
    nslot = 4
    qa, qb = Qrnn(1, 1100, H, ld=H, dev=dev, seed=seed), Qrnn(1, 700, H, ld=H, dev=dev,
                                                               seed=seed + 1)
    wa, wb = [(0, 400), (400, 400), (800, 300)], [(0, 350), (350, 350)]
    # both recordings in one Y / h / Cst: B's rows after A's
    offB = 1100 + 3
    Y = _full((offB + 700) * 3 * H + 64, SENT, dev)
    Y[:1100 * 3 * H] = qa.Y[:1100 * 3 * H]
    Y[offB * 3 * H:(offB + 700) * 3 * H] = qb.Y[:700 * 3 * H]
    h = _full((offB + 716) * H, GUARD, dev)
    Cst = _full((offB + 716) * H, GUARD, dev)
    state = _full(nslot * H, GUARD, dev)
    state[H:2 * H] = SENT
    state[3 * H:4 * H] = SENT
    entering = {}
    for k in range(3):
        a, T = wa[k]
        entering[("A", k)] = state[H:2 * H].clone() if k else torch.zeros(H, device=dev)
        rows = [[a, T, 1, int(k == 0)]]
        if k < 2:
            a, T = wb[k]
            entering[("B", k)] = state[3 * H:4 * H].clone() if k else torch.zeros(H, device=dev)
            rows.append([offB + a, T, 3, int(k == 0)])
        _call(dev, "pase_qrnn_scan_fwd_carry_var", Y, h, H, Cst, state, _i32(rows, dev),
              len(rows), H)
        assert bool((state[:H] == GUARD).all()) and bool((state[2 * H:3 * H] == GUARD).all()), \
            "carry scan wrote another slot"
    out = []
    for q, off, T, slot in ((qa, 0, 1100, 1), (qb, offB, 700, 3)):
        q.h[:T * H] = h[off * H:(off + T) * H]
        q.Cst[:T * H] = Cst[off * H:(off + T) * H]
        assert torch.equal(state[slot * H:(slot + 1) * H], q.Cst[(T - 1) * H:T * H]), \
            "state after the last window != Cst of the last frame"
        out += [("carry fwd T=%d %s" % (T, w), g, r, t) for (w, g, r, t) in qrnn_fwd_checks(q)]
    _unchanged("carry h", h, [(0, 1100 * H), (offB * H, (offB + 700) * H)], GUARD)
    _unchanged("carry Cst", Cst, [(0, 1100 * H), (offB * H, (offB + 700) * H)], GUARD)
    # backward over A's windows, last first; each window has 2 halo frames before its crop
    # (none for the first) and 1 after (none for the last)
    dstate = _full(nslot * H, GUARD, dev)
    dstate[H:2 * H] = 0
    dYs = []
    for k in (2, 1, 0):
        a, cn = wa[k]
        c0 = 0 if k == 0 else 2
        T = c0 + cn + (0 if k == 2 else 1)
        dY = _full((T + 1) * 3 * H + 64, GUARD, dev)
        st = entering[("A", k)]
        sbuf = _full(nslot * H, GUARD, dev)
        sbuf[H:2 * H] = st
        tab = _i32([[a - c0, T, 0, c0, cn, 1]], dev)
        _call(dev, "pase_qrnn_scan_bwd_carry_var", qa.Y, qa.Cst, qa.dh, qa.ld, dY, sbuf, dstate,
              tab, 1, H)
        assert bool((dstate[:H] == GUARD).all()) and bool((dstate[2 * H:] == GUARD).all()), \
            "carry backward wrote another slot"
        dv = dY[:(T + 1) * 3 * H].view(T + 1, 3 * H)
        assert bool((dv[:c0] == 0).all()) and bool((dv[c0 + cn:] == 0).all()), \
            "rows outside the crop not written zero"
        assert bool((dY[(T + 1) * 3 * H:] == GUARD).all()), "carry backward guard"
        dYs.append((a, dv[c0:c0 + cn]))
    for a, d in dYs:
        qa.dY[a * 3 * H:(a + d.shape[0]) * 3 * H] = d.reshape(-1)
    out += [("carry bwd %s" % w, g, r, t) for (w, g, r, t) in qrnn_bwd_checks(qa)]
    return out, (qa, qb, h, Cst, offB, dstate)


def test_qrnn_scan_carry_windows():
    out, (qa, qb, h, Cst, offB, dstate) = qrnn_carry_checks("cuda")
    H = qa.H
    # the forward windows reproduce the whole scan's bits (T' > 512: the sequential kernel);
    # the backward's carried form is held to the float64 bound only, as its header promises
    for q, off, T in ((qa, 0, 1100), (qb, offB, 700)):
        assert _lib.qrnn_scan_plan(T) == 0
        hw, cw = h[off * H:(off + T) * H].clone(), Cst[off * H:(off + T) * H].clone()
        q.h.fill_(GUARD)
        q.Cst.fill_(GUARD)
        q.fwd()
        assert torch.equal(q.h[:T * H], hw) and torch.equal(q.Cst[:T * H], cw), \
            "windowed scan != whole scan (T=%d)" % T
    _report("qrnn carry", _check_all(out))


def test_qrnn_carry_zero_state_round_trip():
    """A zero state and zero dstate: the carried forms are the plain scans of each window."""
    H, T, dev = 64, 600, "cuda"
    q = Qrnn(1, T, H, ld=H, dev=dev, seed=70)
    state = torch.zeros(2 * H, device=dev)
    _call(dev, "pase_qrnn_scan_fwd_carry_var", q.Y, q.h, H, q.Cst, state, _i32([[0, T, 1, 0]], dev),
          1, H)
    assert torch.equal(state[H:], q.Cst[(T - 1) * H:T * H])
    r = qrnn_fwd_checks(q)
    dstate = torch.zeros(2 * H, device=dev)
    dstate[:H] = GUARD
    st0 = torch.zeros(2 * H, device=dev)
    dY = _full((T + 1) * 3 * H, GUARD, dev)
    _call(dev, "pase_qrnn_scan_bwd_carry_var", q.Y, q.Cst, q.dh, q.ld, dY, st0, dstate,
          _i32([[0, T, 0, 0, T, 1]], dev), 1, H)
    q.dY[:T * 3 * H] = dY[:T * 3 * H]
    assert bool((dY[T * 3 * H:] == 0).all())
    r += qrnn_bwd_checks(q)
    # dstate: the gradient of the entering state, dc_0 (1 - f_0), with dc_0 and its bound from
    # the recurrence of qrnn_bwd_checks
    y = q.Y[:T * 3 * H].view(T, 3, H).double()
    f, o = torch.sigmoid(y[:, 1]), torch.sigmoid(y[:, 2])
    g = q.hview(q.dh)[0].double()
    carry, eps, M = (torch.zeros(H, dtype=torch.float64, device=dev) for _ in range(3))
    a_next = torch.zeros_like(carry)
    for t in range(T - 1, -1, -1):
        go = g[t] * o[t]
        dc = go + carry
        eps = a_next * eps + K_QRNN * U * (go.abs() + M)
        M = go.abs() + a_next * M
        a_next = 1.0 - f[t]
        carry = dc * a_next
    assert bool((dstate[:H] == GUARD).all()), "dstate: another slot written"
    dc0 = carry / a_next.clamp_min(1e-300)
    # 1 - f is off by 6u f + u (1 - f) (saturated gates: exactly 0 in fp32)
    tol = (eps + K_QRNN * U * M) * a_next + U * carry.abs() \
        + (dc0.abs() + eps) * (6 * U * f[0] + U * a_next)
    r.append(("dstate", dstate[H:], carry, tol))
    _report("qrnn carry zero state", _check_all(r))


# ================================ output layer ================================
class OutVar(object):
    def __init__(self, Ts, C, dev, gap=2, seed=0):
        self.Ts, self.C, self.dev = list(Ts), C, dev
        gen = torch.Generator().manual_seed(5500 + seed)
        n = len(Ts)
        self.row0 = np.concatenate([[0], np.cumsum(np.asarray(Ts) + gap)])[:n]
        rows = int(self.row0[-1] + Ts[-1] + gap)
        y = torch.full((rows * C,), SENT)
        for r0, T in zip(self.row0, Ts):
            y[r0 * C:(r0 + T) * C] = torch.randn(T * C, generator=gen) * 2.0 + 0.7
        self.y = y.to(dev)
        self.scale = torch.randn(C, generator=gen).to(dev)
        self.shift = torch.randn(C, generator=gen).to(dev)
        self.mean = (torch.randn(C, generator=gen) * 0.5).to(dev)
        self.invstd = (torch.randn(C, generator=gen).abs() + 0.5).to(dev)
        self.rows = rows
        self.gen = gen

    def h(self, i):
        r0, T = int(self.row0[i]), self.Ts[i]
        return self.y[r0 * self.C:(r0 + T) * self.C].view(T, self.C).double() \
            * self.scale.double() + self.shift.double()


def out_affine_var_checks(o, mode):
    C, n = o.C, len(o.Ts)
    E_ = C * (2 if mode >= 2 else 1)
    offs = np.concatenate([[0], np.cumsum(E_ * np.asarray(o.Ts) + 3)])[:n]
    out = _full(int(offs[-1] + E_ * o.Ts[-1] + 3), GUARD, o.dev)
    tab = _i32(np.stack([o.row0, o.Ts, offs], 1), o.dev)
    _call(o.dev, "pase_out_affine_var", o.y, o.scale, o.shift, out, tab, n, C, mode)
    checks, spans = [], []
    for i, T in enumerate(o.Ts):
        h = o.h(i).t()                                   # (C, T)
        m = h.mean(1, keepdim=True)
        hm = h.abs().max(1, keepdim=True).values
        mt = 1e-6 * hm
        parts = {0: [(h, _ulp32(h))], 1: [(h - m, _ulp32(h) + mt + _ulp32(h - m))],
                 2: [(h, _ulp32(h)), (m.expand(C, T), mt.expand(C, T))],
                 3: [(h - m, _ulp32(h) + mt + _ulp32(h - m)), (m.expand(C, T), mt.expand(C, T))]}
        got = out[int(offs[i]):int(offs[i]) + E_ * T].view(E_, T)
        for k, (ref, tol) in enumerate(parts[mode]):
            checks.append(("out mode %d utt %d part %d" % (mode, i, k), got[k * C:(k + 1) * C],
                           ref, tol))
        spans.append((int(offs[i]), int(offs[i]) + E_ * T))
    _unchanged("out", out, spans, GUARD)
    return checks


def out_place_select_checks(o, mode):
    """pase_out_place_var windows of two streams (rows alternate) into a (C, ld) block each at
    its own ocol, then pase_out_select over a whole (C, T) output."""
    C, n = o.C, len(o.Ts)
    ld = sum(o.Ts) + 5
    out = _full(2 * C * ld + 64, GUARD, o.dev)
    col0 = np.concatenate([[0], np.cumsum(o.Ts)])[:n] + 2
    ocol = (np.arange(n) % 2) * ld                 # stream 1's block starts at element ld * C
    tab = _i32(np.stack([o.row0, o.Ts, ocol, np.full(n, ld), col0], 1), o.dev)
    _call(o.dev, "pase_out_place_var", o.y, o.scale, o.shift, out, tab, n, max(o.Ts), C)
    checks, spans = [], []
    for i, T in enumerate(o.Ts):
        h = o.h(i).t()
        b0 = int(ocol[i]) * C
        blk = out[b0:b0 + C * ld].view(C, ld)
        checks.append(("place %d" % i, blk[:, int(col0[i]):int(col0[i]) + T], h, _ulp32(h)))
        spans += [(b0 + c * ld + int(col0[i]), b0 + c * ld + int(col0[i]) + T) for c in range(C)]
    _unchanged("place out", out, spans, GUARD)
    # select_output over a whole (C, T) output of T = sum Ts frames, rows C..2C-1 for the mean
    T = sum(o.Ts)
    h = torch.cat([o.h(i).t() for i in range(n)], 1)
    buf = _full(2 * C * T + 16, GUARD, o.dev)
    buf[:C * T] = h.float().reshape(-1)
    h32 = buf[:C * T].view(C, T).double()
    _call(o.dev, "pase_out_select", buf, T, C, mode)
    m = h32.mean(1, keepdim=True)
    mt = 1e-6 * h32.abs().max(1, keepdim=True).values
    got = buf[:2 * C * T].view(2 * C, T) if mode >= 2 else buf[:C * T].view(C, T)
    if mode in (1, 3):
        checks.append(("select norm", got[:C], h32 - m, mt + _ulp32(h32 - m)))
    else:
        assert torch.equal(got[:C], h32.float()), "select changed h"
    if mode >= 2:
        checks.append(("select mean", got[C:], m.expand(C, T), mt.expand(C, T)))
    _unchanged("select", buf, [(0, (2 if mode >= 2 else 1) * C * T)], GUARD)
    return checks


def out_bwd_checks(o, dev=None):
    """pase_out_bwd_gather_var (exact), pase_out_bwd_reduce_var (exact gather, S1 / S2 within
    2^-16) and pase_out_bwd_gather_crop (exact, zeros outside the crop)."""
    C, n, dev = o.C, len(o.Ts), o.dev
    o_off = np.concatenate([[0], np.cumsum(C * np.asarray(o.Ts) + 3)])[:n]
    dout = torch.full((int(o_off[-1] + C * o.Ts[-1] + 3),), SENT)
    for a, T in zip(o_off, o.Ts):
        dout[a:a + C * T] = torch.randn(C * T, generator=o.gen)
    dout = dout.to(dev)
    tab = _i32(np.stack([o.row0, o.Ts, o_off], 1), dev)
    g = _full(o.rows * C, GUARD, dev)
    _call(dev, "pase_out_bwd_gather_var", dout, tab, n, max(o.Ts), C, g)
    g2 = _full(o.rows * C, GUARD, dev)
    S1, S2 = (_full(C + 4, GUARD, dev, torch.float64) for _ in range(2))
    S1[:C] = 0
    S2[:C] = 0
    _call(dev, "pase_out_bwd_reduce_var", dout, tab, n, max(o.Ts), C, o.y, o.mean, o.invstd, g2,
          S1, S2)
    spans = []
    s1 = torch.zeros(C, dtype=torch.float64, device=dev)
    s2, m1, m2 = s1.clone(), s1.clone(), s1.clone()
    for i, T in enumerate(o.Ts):
        r0, a = int(o.row0[i]), int(o_off[i])
        ref = dout[a:a + C * T].view(C, T).t()
        assert torch.equal(g[r0 * C:(r0 + T) * C].view(T, C), ref), "gather not exact"
        assert torch.equal(g2[r0 * C:(r0 + T) * C].view(T, C), ref), "reduce gather not exact"
        spans.append((r0 * C, (r0 + T) * C))
        xh = (o.y[r0 * C:(r0 + T) * C].view(T, C).double() - o.mean.double()) \
            * o.invstd.double()
        s1 += ref.double().sum(0)
        m1 += ref.double().abs().sum(0)
        s2 += (ref.double() * xh).sum(0)
        m2 += (ref.double() * xh).abs().sum(0)
    _unchanged("g_ntc", g, spans, GUARD)
    _unchanged("g_ntc (reduce)", g2, spans, GUARD)
    assert bool((S1[C:] == GUARD).all()) and bool((S2[C:] == GUARD).all())
    checks = [("S1", S1[:C], s1, 2.0 ** -16 * m1), ("S2", S2[:C], s2, 2.0 ** -16 * m2)]
    # the crop of a (C, ld) recording gradient
    ld, col0, T, c0, cn = 1000, 333, 120, 7, 100
    rec = torch.randn(C * ld, generator=o.gen).to(dev)
    gc = _full(T * C + 16, GUARD, dev)
    _call(dev, "pase_out_bwd_gather_crop", rec, ld, col0, T, c0, cn, C, gc)
    ref = torch.zeros(T, C, device=dev)
    ref[c0:c0 + cn] = rec.view(C, ld)[:, col0:col0 + cn].t()
    assert torch.equal(gc[:T * C].view(T, C), ref), "gather_crop not exact"
    assert bool((gc[T * C:] == GUARD).all()), "gather_crop guard"
    return checks


def stream_gather_checks(dev):
    """Two rows whose ring reads and appends wrap around ring_cap; slot 0 untouched."""
    cap, gen = 1000, torch.Generator().manual_seed(5600)
    ring = torch.randn(3 * cap, generator=gen).to(dev)
    staging = torch.randn(400, generator=gen).to(dev)
    wave = _full(420, GUARD, dev)
    rows = [[1, 900, 250, 0, 700, 200, 300, 0],       # append 900..1149 (wraps), read 700..899
            [2, 10, 30, 250, 950, 60, 90, 310]]       # read 950..1009 (wraps), append 10..39
    ring0 = ring.clone()
    _call(dev, "pase_stream_gather", staging, ring, cap, wave, _i32(rows, dev), 2, 300)
    r1, r2 = ring0[cap:2 * cap], ring0[2 * cap:]
    exp1 = torch.cat([r1[700:900], staging[:100]])
    exp2 = torch.cat([r2[950:], r2[:10], staging[250:280]])
    assert torch.equal(wave[:300], exp1) and torch.equal(wave[310:400], exp2), "gathered segment"
    _unchanged("wave", wave, [(0, 300), (310, 400)], GUARD)
    n1, n2 = r1.clone(), r2.clone()
    n1[900:] = staging[:100]
    n1[:150] = staging[100:250]
    n2[10:40] = staging[250:280]
    assert torch.equal(ring[:cap], ring0[:cap]), "slot 0 written"
    assert torch.equal(ring[cap:2 * cap], n1) and torch.equal(ring[2 * cap:], n2), "ring append"


OUT_TS = [1, 25, 300, 513, 3]


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_out_affine_var(mode):
    o = OutVar(OUT_TS, 256, "cuda", seed=mode)
    r = out_affine_var_checks(o, mode)
    if mode == 0:                 # bits of pase_out_affine_nct at N = 1
        for i, T in enumerate(OUT_TS):
            o1 = _full(256 * T, 0.0, "cuda")
            _call("cuda", "pase_out_affine_nct", o.y[int(o.row0[i]) * 256:], o.scale, o.shift, o1,
                  None, 1, T, 256)
            assert torch.equal(o1.view(256, T), r[i][1]), "packed != pase_out_affine_nct"
    _report("out_affine_var mode %d" % mode, _check_all(r))


@pytest.mark.parametrize("mode", [1, 2, 3])
def test_out_place_and_select(mode):
    o = OutVar(OUT_TS, 100, "cuda", seed=10 + mode)
    _report("out place/select mode %d" % mode, _check_all(out_place_select_checks(o, mode)))


def test_out_bwd_var_and_crop():
    o = OutVar(OUT_TS, 256, "cuda", seed=20)
    _report("out bwd var", _check_all(out_bwd_checks(o)))


def test_stream_gather_ring_wrap():
    stream_gather_checks("cuda")


# ================================ 64-bit offsets ================================
def test_64bit_offsets():
    """One buffer of just over 2^31 fp32 elements shared by pase_out_place_var (ocol C > 2^31),
    pase_out_bwd_gather_crop (col0 C-scale offsets) and pase_reflect_fold_wave_acc
    (x0 > 2^31); only the touched windows and a guard band on each side are checked."""
    free = torch.cuda.mem_get_info()[0]
    if free < 12 * 2 ** 30:
        print("64-bit offsets: skipped, %.1f GB free < 12 GB" % (free / 2 ** 30))
        pytest.skip("needs 12 GB free")
    n = 2 ** 31 + 2 ** 20
    buf = torch.empty(n, dtype=torch.float32, device="cuda")
    try:
        band = 4096
        # out_place_var: C = 4, ocol * C just past 2^31
        C, T, ld, c0 = 4, 37, 64, 5
        ocol = (2 ** 31 + 1000) // C
        base = ocol * C
        assert base > 2 ** 31 and base + C * ld < n
        buf[base - band:base + C * ld + band] = GUARD
        gen = torch.Generator(device="cuda").manual_seed(64)
        y = torch.randn(T * C, generator=gen, device="cuda")
        sc, sh = torch.randn(C, generator=gen, device="cuda"), torch.randn(C, device="cuda")
        _call("cuda", "pase_out_place_var", y, sc, sh, buf, _i32([[0, T, ocol, ld, c0]], "cuda"),
              1, T, C)
        blk = buf[base:base + C * ld].view(C, ld)
        ref = (y.view(T, C).double() * sc.double() + sh.double()).t()
        _within("place 64-bit", blk[:, c0:c0 + T], ref, _ulp32(ref))
        win = buf[base - band:base + C * ld + band].clone()
        keep = torch.ones_like(win, dtype=torch.bool)
        torch.as_strided(keep, (C, T), (ld, 1), band + c0).fill_(False)
        assert bool((win[keep] == GUARD).all()), "place 64-bit: guard written"
        # gather_crop: the buffer as a (C, ld2) recording gradient, offsets c*ld2 + col0 > 2^31
        C2 = 4
        ld2 = n // C2
        col0, Tc, cc0, cn = ld2 - 300, 200, 3, 150
        for c in range(C2):
            buf[c * ld2 + col0:c * ld2 + col0 + cn] = torch.arange(cn, device="cuda") + 1000 * c
        g = _full(Tc * C2 + 16, GUARD, "cuda")
        _call("cuda", "pase_out_bwd_gather_crop", buf, ld2, col0, Tc, cc0, cn, C2, g)
        refc = torch.zeros(Tc, C2, device="cuda")
        refc[cc0:cc0 + cn] = (torch.arange(cn, device="cuda")[:, None]
                              + 1000 * torch.arange(C2, device="cuda")[None, :]).float()
        assert torch.equal(g[:Tc * C2].view(Tc, C2), refc), "gather_crop 64-bit"
        assert bool((g[Tc * C2:] == GUARD).all())
        # fold_acc: x0 > 2^31
        x0, Tw, pL, pR = 2 ** 31 + 12345, 3000, 125, 125
        buf[x0 - band:x0 + Tw + band] = GUARD
        buf[x0:x0 + Tw] = 0.0
        d = torch.randn(Tw + pL + pR, generator=gen, device="cuda")
        _call("cuda", "pase_reflect_fold_wave_acc", d, buf, x0, Tw, pL, pR, 1, 1)
        idx = emul.core._reflect(torch.arange(Tw + pL + pR) - pL, Tw).cuda()
        refd = torch.zeros(Tw, dtype=torch.float64, device="cuda").index_add_(0, idx, d.double())
        mag = torch.zeros(Tw, dtype=torch.float64, device="cuda").index_add_(
            0, idx, d.double().abs())
        _within("fold_acc 64-bit", buf[x0:x0 + Tw], refd, 2 * U * mag)
        assert bool((buf[x0 - band:x0] == GUARD).all()) and \
            bool((buf[x0 + Tw:x0 + Tw + band] == GUARD).all()), "fold_acc 64-bit: guard"
        print("64-bit offsets: place at %d, crop up to %d, fold at %d" %
              (base, (C2 - 1) * ld2 + col0, x0))
    finally:
        del buf
        torch.cuda.empty_cache()


# ================================ refusals ================================
def _dummy(dev="cuda"):
    f = lambda n: torch.zeros(n, device=dev)
    i = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)
    d = lambda n: torch.zeros(n, dtype=torch.float64, device=dev)
    return f, i, d


def _grid_row_calls(nseg):
    """Every entry point with a grid row per utterance, called with `nseg` rows and otherwise
    valid arguments (the table is large enough for 65535 rows of the widest entry)."""
    f, i, d = _dummy()
    tab = i(9 * 65536)
    x, C, H = f(4096), 8, 8
    return {
        "pase_reflect_pad_wave_var": (x, tab, nseg, 4, x, None, 0, 1, 1),
        "pase_reflect_fold_wave_var": (x, tab, nseg, 4, x, 1, 1),
        "pase_bn_prelu_pad_fwd_var": (x, 0, tab, nseg, 4, C, f(C), f(C), f(C), x, None, 0, C, 0,
                                      0, None, C, 0),
        "pase_bn_prelu_bwd_reduce_var": (x, 0, tab, nseg, 4, C, f(C), f(C), f(C), f(C), f(C), x,
                                         0, C, 0, 0, None, C, 0, None, C, d(C), d(C), d(C), None),
        "pase_bn_prelu_bwd_apply_src_var": (x, 0, tab, nseg, 4, C, f(C), f(C), f(C), f(C), f(C),
                                            x, 0, C, 0, 0, None, C, 0, None, C, x, None, 0, 0,
                                            None, None, None),
        "pase_bn_prelu_bwd_apply_src_var_train": (x, 0, tab, nseg, 4, C, f(C), f(C), f(C), f(C),
                                                  f(C), f(C), d(C), d(C), 1.0, x, 0, C, 0, 0,
                                                  None, C, 0, None, C, x, None, 0, 0, None, None,
                                                  None),
        "pase_out_affine_var": (x, f(C), f(C), x, tab, nseg, C, 0),
        "pase_out_place_var": (x, f(C), f(C), x, tab, nseg, 4, C),
        "pase_out_bwd_gather_var": (x, tab, nseg, 4, C, x),
        "pase_out_bwd_reduce_var": (x, tab, nseg, 4, C, x, f(C), f(C), x, d(C), d(C)),
        "pase_qrnn_scan_fwd_var": (x, x, H, x, tab, nseg, H),
        "pase_qrnn_scan_bwd_var": (x, x, x, H, x, tab, nseg, H),
        "pase_qrnn_scan_fwd_carry_var": (x, x, H, x, x, tab, nseg, H),
        "pase_qrnn_scan_bwd_carry_var": (x, x, x, H, x, x, x, tab, nseg, H),
        "pase_stream_gather": (x, x, 16, x, tab, nseg, 4),
    }


GRID_ROW_ENTRIES = [
    "pase_reflect_pad_wave_var", "pase_reflect_fold_wave_var", "pase_bn_prelu_pad_fwd_var",
    "pase_bn_prelu_bwd_reduce_var", "pase_bn_prelu_bwd_apply_src_var",
    "pase_bn_prelu_bwd_apply_src_var_train", "pase_out_affine_var", "pase_out_place_var",
    "pase_out_bwd_gather_var", "pase_out_bwd_reduce_var", "pase_qrnn_scan_fwd_var",
    "pase_qrnn_scan_bwd_var", "pase_qrnn_scan_fwd_carry_var", "pase_qrnn_scan_bwd_carry_var",
    "pase_stream_gather"]


@pytest.mark.parametrize("name", GRID_ROW_ENTRIES)
def test_refuses_more_grid_rows_than_the_launch_holds(name):
    """nseg = 65536 (one past gridDim.y's limit) and nseg = 0 are refused before any launch."""
    for nseg in (MAX_GRID_Y + 1, 0):
        with pytest.raises(RuntimeError, match=name + r"\b.*(nseg|nrow|bad args)"):
            _lib.call(name, *_grid_row_calls(nseg)[name])
    torch.cuda.synchronize()


@pytest.mark.parametrize("name,args,pattern", [
    ("pase_out_bwd_gather_crop", dict(c0=60, cn=50), "bad args"),        # crop past T
    ("pase_out_bwd_gather_crop", dict(col0=990, cn=20), "bad args"),     # past ld
    ("pase_out_bwd_gather_crop", dict(c0=-1), "bad args"),
    ("pase_out_bwd_gather_crop", dict(cn=0), "bad args"),
    ("pase_out_select", dict(mode=0), "mode 0"),
    ("pase_out_affine_var", dict(mode=4), "mode 4"),
    ("pase_reflect_fold_wave_acc", dict(x0=-1), "bad args"),
    ("pase_reflect_fold_wave_acc", dict(padL=100), "bad args"),         # pad >= T
    ("pase_reflect_fold_wave_acc", dict(padR=100), "bad args"),
    ("pase_stream_gather", dict(max_len=17), "max_len=17 past ring_cap"),
    ("pase_stream_gather", dict(ring_cap=0), "ring_cap=0"),
])
def test_documented_refusals(name, args, pattern):
    f, i, d = _dummy()
    base = {
        "pase_out_bwd_gather_crop": dict(dout=f(8000), ld=1000, col0=0, T=100, c0=0, cn=10, C=8,
                                         g_ntc=f(800)),
        "pase_out_select": dict(out=f(800), T=50, C=8, mode=1),
        "pase_out_affine_var": dict(y=f(80), scale=f(8), shift=f(8), out=f(80),
                                    tab=i(3), nseg=1, C=8, mode=0),
        "pase_reflect_fold_wave_acc": dict(dpad=f(300), dx=f(200), x0=0, T=100, padL=10,
                                           padR=10, fold_l=1, fold_r=1),
        "pase_stream_gather": dict(staging=f(64), ring=f(64), ring_cap=16, wave=f(64),
                                   tab=i(8), nrow=1, max_len=4),
    }[name]
    names = [p for (_, _, p) in _lib.PROTOS[name][1] if p != "stream"]
    _lib.call(name, *[base[p] for p in names])
    torch.cuda.synchronize()
    base.update(args)
    with pytest.raises(RuntimeError, match=name + ".*" + pattern):
        _lib.call(name, *[base[p] for p in names])
