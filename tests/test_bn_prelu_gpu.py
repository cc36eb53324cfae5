"""The BatchNorm + PReLU kernels (pase_bn_prelu_pad_fwd, pase_bn_prelu_bwd_reduce,
pase_bn_prelu_bwd_apply, pase_bn_prelu_bwd_apply_src) against a float64 reference computed
with torch on the device directly from the fp32 / bf16 inputs, in the regimes the training
step runs them.

Every backward case asserts which kernel it reaches through pase_bn_bwd_plan (using the
device's SM count) and prints the plan.  The staged cases give some block more than STAGES
tiles for any SM count up to 132 (the ring wraps, the mbarrier parity flips, the pooled
gradient is prefetched a tile ahead and a block's tiles cross from one sample into the next);
the grid-stride cases give every thread more than one run.

Memory the kernels must not read (slack rows and columns of y, srcA, srcB and pool) holds a
huge finite sentinel, so a stray read shows up as a large error; memory they must not write
(guard elements around dst / dst_lo / du and pool columns) is checked unchanged.

Bounds (u = 2^-24):
  sums S1 / S2 / dalpha / db: 2^-16 x the per-channel sum of the terms' magnitudes;
  fp32 du / dy: 2^-20 x |gamma invstd| (|du| + |S1/M| + |xhat| |S2/M|), where |du| counts
    the magnitudes of the gradient sources it sums (each fp32 addition rounds relative to
    them) and S1 / S2 are fed identically to kernel and reference;
  bf16: one bf16 ulp of the reference (plus the fp32 bound);  fp16 pair: hi + lo/2^11
    against s x ref at 2^-21 of the bound more, scale_out bit-exact;
  tf32 residual twin: trunc_tf32(dst) + lo == dst to 2^-21 and lo == residual(dst) exactly;
  forward: dst within 2 fp32 ulps; a pooling window mean, summed in fp32 over pool_d steps,
    within (pool_d + 4) u x mean|a| (the worst-case error of that sum).
The PReLU gate is kept unambiguous: every y with |y*scale + shift| < 1e-3 |scale| is moved
away from the kink, so an fp32 rounding cannot flip a gate."""
import pytest
import torch

import emul            # bit-level operand formats only (tf32 residual, fp16 gradient scale)
from pase_b200 import _lib
from pase_b200 import encoder as E

pytestmark = pytest.mark.gpu

THREADS = 256              # threads per block of every BatchNorm/PReLU kernel
STAGES = 3                 # depth of the staged kernels' shared-memory ring
MAX_SMS = 132              # the cases hold their regime for any SM count up to this
SENT = 2.0 ** 100          # huge finite sentinel in memory the kernels must not read
GUARD = {torch.float32: 2.0 ** 100, torch.bfloat16: 2.0 ** 100, torch.float16: 2.0 ** 15}
U = 2.0 ** -24

# (y bf16, srcA bf16, dst format, tf32 / fp16 low twin) of each encoder precision
PRECS = {"fp32": (0, 0, 0, False), "3xtf32": (0, 0, 0, True), "bf16": (1, 1, 1, False),
         "bf16-a32": (1, 0, 1, False), "3xf16": (0, 0, 2, True)}
FMT_DTYPE = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}


def _view(buf, shape, strides, off=0):
    return torch.as_strided(buf, shape, strides, buf.storage_offset() + off)


def _randn(n, gen, scale=1.0):
    return torch.randn(int(n), generator=gen, device="cuda", dtype=torch.float32) * scale


def _ulp(x, mant):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - mant)


def _within(what, got, ref, tol):
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err - tol, torch.zeros_like(err)).reshape(-1)))
        raise AssertionError("%s: %d/%d out of bound; worst at flat %d: got %.9e ref %.9e "
                             "err %.3e tol %.3e" % (what, int(bad.sum()), bad.numel(), i,
                                                    float(got.reshape(-1)[i]),
                                                    float(ref.reshape(-1)[i]),
                                                    float(err.reshape(-1)[i]),
                                                    float(tol.reshape(-1)[i])))


def _untouched(what, buf, shape, strides, off=0):
    """Every element of buf outside the strided view still holds its guard value."""
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    _view(keep, shape, strides, off).fill_(False)
    rest = buf[keep]
    assert torch.equal(rest, torch.full_like(rest, GUARD[buf.dtype])), what + ": guard written"


def _guarded(n, dtype):
    return torch.full((int(n),), GUARD[dtype], dtype=dtype, device="cuda")


def _bn_params(C, gen):
    p = dict(mean=_randn(C, gen, 0.1), invstd=_randn(C, gen).abs() + 0.5, gamma=_randn(C, gen),
             scale=_randn(C, gen), shift=_randn(C, gen, 0.5), alpha=_randn(C, gen, 0.3))
    return p


def _make_y(N, T, C, y_ss, ybf, p, gen):
    """y (N, T, C) at sample stride y_ss in its storage type, sentinel in the slack, every
    value at least 1e-3 away from its channel's PReLU kink."""
    dt = torch.bfloat16 if ybf else torch.float32
    y = torch.full((N * y_ss + 64,), SENT, dtype=dt, device="cuda")
    v = _randn(N * T * C, gen).view(N, T, C)
    kink = -p["shift"].double() / p["scale"].double()
    for step in (0.05, 0.2, 1.0, None):
        v = v.to(dt).float()                   # the value the kernel reads
        near = (v.double() - kink).abs() < 1e-3
        if not bool(near.any()):
            break
        assert step is not None, "could not move y away from the PReLU kink"
        away = torch.where(v.double() >= kink, 1.0, -1.0)
        v = torch.where(near, (kink + away * step).float(), v)
    _view(y, (N, T, C), (y_ss, C, 1)).copy_(v.to(dt))
    return y


class Bwd(object):
    """Operands of one backward call pair (pass 1 sums, pass 2 dy) and the results."""

    def __init__(self, N, T, C, prec="fp32", padL=0, padR=0, a_rs=None, a_ss=None,
                 interleaved=False, pool_d=0, pool_T=None, p_rs=None, p_ss=None, p_off=0,
                 y_ss=None, d_ss=None, doff=0, dbias=True, train=True, priors=False, du=False,
                 seed=0):
        gen = torch.Generator(device="cuda").manual_seed(1000 + seed)
        self.N, self.T, self.C, self.prec = N, T, C, prec
        self.ybf, self.abf, self.fmt, lo = PRECS[prec]
        self.train, self.stored_du = train, du
        self.p = _bn_params(C, gen)
        self.y_ss = y_ss if y_ss is not None else T * C
        self.y = _make_y(N, T, C, self.y_ss, self.ybf, self.p, gen)
        # gradient source A (+ B): the next layer's padded input gradient, or the PASE+ last
        # block's interleaved [x_{t-1} | x_t] QRNN input gradient (A = dsrc[C:], B = dsrc)
        adt = torch.bfloat16 if self.abf else torch.float32
        self.padL, self.padR = padL, padR
        Tp = T + padL + padR
        if interleaved:
            assert padL == 0 and padR == 0 and not self.abf
            self.a_rs = self.b_rs = 2 * C
            self.a_ss = self.b_ss = T * 2 * C
            D = _randn(N * T * 2 * C, gen)
            _view(D, (N, C), (T * 2 * C, 1)).fill_(SENT)      # B row 0: never read (shift 1)
            self.Abuf, self.A, self.B, self.b_shift = D, D[C:], D, 1
        else:
            self.a_rs = a_rs if a_rs is not None else C
            self.a_ss = a_ss if a_ss is not None else (Tp + 1) * self.a_rs
            self.Abuf = torch.full((N * self.a_ss + self.a_rs,), SENT, dtype=adt, device="cuda")
            _view(self.Abuf, (N, Tp, C), (self.a_ss, self.a_rs, 1)).copy_(
                _randn(N * Tp * C, gen).view(N, Tp, C).to(adt))
            self.A, self.B, self.b_ss, self.b_rs, self.b_shift = self.Abuf, None, 0, 0, 0
        # mean-pooled dense-skip gradient: columns C.. of a wide concat pitch belong to the
        # other blocks
        self.pool_d = pool_d
        self.pool_T = pool_T if pool_T is not None else (T // pool_d if pool_d else 0)
        if pool_d:
            self.p_rs = p_rs if p_rs is not None else C + 64
            self.p_ss = p_ss if p_ss is not None else (self.pool_T + 1) * self.p_rs
            self.Pbuf = torch.full((p_off + N * self.p_ss + self.p_rs,), SENT, device="cuda")
            self.P = self.Pbuf[p_off:]
            _view(self.P, (N, self.pool_T, C), (self.p_ss, self.p_rs, 1)).copy_(
                _randn(N * self.pool_T * C, gen).view(N, self.pool_T, C))
        else:
            self.p_rs = self.p_ss = 0
            self.P = None
        # outputs: dy (format fmt, + low twin) at sample stride d_ss from offset doff
        self.d_ss = d_ss if d_ss is not None else T * C
        self.doff = doff
        odt = FMT_DTYPE[self.fmt]
        n_out = doff + N * self.d_ss + 64
        self.dst_buf = _guarded(n_out, odt)
        self.lo_buf = _guarded(n_out, odt) if lo else None
        self.du_buf = _guarded(n_out, self.y.dtype) if du else None
        f64 = dict(dtype=torch.float64, device="cuda")
        self.prior = {k: (torch.randn(C, generator=gen, device="cuda", dtype=torch.float64) * 10
                          if priors else torch.zeros(C, **f64)) for k in ("S1", "S2", "dal", "db")}
        self.S1, self.S2, self.dal = (self.prior[k].clone() for k in ("S1", "S2", "dal"))
        self.db = self.prior["db"].clone() if dbias else None
        use_amax = self.fmt == 2 or priors
        self.amax_prior = torch.tensor([1e-3, 100.0] if priors else [0.0, 0.0], device="cuda")
        self.amax = self.amax_prior.clone() if use_amax else None
        self.scale_out = torch.zeros(2, device="cuda") if self.fmt == 2 else None

    def src(self):
        return (self.A, self.abf, self.a_ss, self.a_rs, self.padL, self.padR, self.B, self.b_ss,
                self.b_rs, self.b_shift, self.P, self.p_ss, self.p_rs, self.pool_d, self.pool_T)

    def head(self):
        return (self.y, self.ybf, self.y_ss, self.N, self.T, self.C)

    def out(self, buf):
        return None if buf is None else buf[self.doff:]

    def plans(self):
        p1 = _lib.bn_bwd_plan(1, *self.head(), *self.src(), self.out(self.du_buf), None, 0,
                              self.d_ss)
        src2 = (None, 0, 0, 0, 0, 0, None, 0, 0, 0, None, 0, 0, 0, 0) if self.stored_du \
            else self.src()
        p2 = _lib.bn_bwd_plan(2, *self.head(), *src2, self.out(self.dst_buf),
                              self.out(self.lo_buf), self.fmt, self.d_ss)
        return p1, p2

    def run(self):
        p, M = self.p, float(self.N * self.T)
        _lib.call("pase_bn_prelu_bwd_reduce", *self.head(), p["mean"], p["invstd"], p["scale"],
                  p["shift"], p["alpha"], *self.src(), self.out(self.du_buf), self.d_ss, self.S1,
                  self.S2, self.dal, self.amax)
        zero = torch.zeros(self.C, dtype=torch.float64, device="cuda")
        self.S1in, self.S2in = (self.S1, self.S2) if self.train else (zero, zero.clone())
        amax2 = self.amax if self.fmt == 2 else None
        if self.stored_du:
            _lib.call("pase_bn_prelu_bwd_apply", *self.head(), p["mean"], p["invstd"],
                      p["gamma"], self.S1in, self.S2in, M, self.out(self.du_buf),
                      self.out(self.dst_buf), self.out(self.lo_buf), self.fmt, self.d_ss,
                      self.db, amax2, self.scale_out)
        else:
            _lib.call("pase_bn_prelu_bwd_apply_src", *self.head(), p["mean"], p["invstd"],
                      p["gamma"], p["scale"], p["shift"], p["alpha"], self.S1in, self.S2in, M,
                      *self.src(), self.out(self.dst_buf), self.out(self.lo_buf), self.fmt,
                      self.d_ss, self.db, amax2, self.scale_out)
        torch.cuda.synchronize()


def _bwd_reference(b):
    """float64: summed gradient sources g (and the sum of their magnitudes), u, the gate, du,
    xhat and the pass-1 sums."""
    N, T, C, p = b.N, b.T, b.C, b.p
    y = _view(b.y, (N, T, C), (b.y_ss, C, 1)).double()
    Tp = T + b.padL + b.padR
    a = _view(b.A, (N, Tp, C), (b.a_ss, b.a_rs, 1)).double()
    idx = (torch.arange(Tp, device="cuda") - b.padL).abs()
    idx = torch.where(idx >= T, 2 * (T - 1) - idx, idx)           # reflect fold-back
    g = torch.zeros(N, T, C, dtype=torch.float64, device="cuda")
    gabs = torch.zeros_like(g)
    g.index_add_(1, idx, a)
    gabs.index_add_(1, idx, a.abs())
    if b.B is not None:                                            # shifted second source
        bv = _view(b.B, (N, T, C), (b.b_ss, b.b_rs, 1)).double()
        s = b.b_shift
        g[:, :T - s] += bv[:, s:]
        gabs[:, :T - s] += bv[:, s:].abs()
    if b.P is not None and b.pool_d > 0:                           # pooled broadcast
        L = b.pool_T * b.pool_d
        pv = _view(b.P, (N, b.pool_T, C), (b.p_ss, b.p_rs, 1)).double() / b.pool_d
        pv = pv.repeat_interleave(b.pool_d, dim=1)
        g[:, :L] += pv
        gabs[:, :L] += pv.abs()
    u = y * p["scale"].double() + p["shift"].double()
    pos = u > 0
    gate = torch.where(pos, 1.0, p["alpha"].double().expand(N, T, C))
    du = gate * g
    duabs = gate.abs() * gabs
    xh = (y - p["mean"].double()) * p["invstd"].double()
    zero = torch.zeros_like(g)
    return dict(g=g, du=du, duabs=duabs, xh=xh,
                S1=du.sum((0, 1)), S1abs=duabs.sum((0, 1)),
                S2=(du * xh).sum((0, 1)), S2abs=(duabs * xh.abs()).sum((0, 1)),
                dal=torch.where(pos, zero, u * g).sum((0, 1)),
                dalabs=torch.where(pos, zero, u.abs() * gabs).sum((0, 1)))


def _check_bwd(b, r):
    N, T, C, p = b.N, b.T, b.C, b.p
    for k, got in (("S1", b.S1), ("S2", b.S2), ("dal", b.dal)):
        pr = b.prior[k]
        _within("pass 1 " + k, got, pr + r[k], 2.0 ** -16 * r[k + "abs"] + 2.0 ** -40 * pr.abs())
    if b.amax is not None:
        ref = torch.stack([r["du"].abs().max(), r["xh"].abs().max()])
        ref = torch.maximum(ref, b.amax_prior.double())
        _within("amax", b.amax, ref, 2.0 ** -20 * torch.stack([r["duabs"].max(), ref[1]]))
    if b.stored_du:
        du = _view(b.out(b.du_buf), (N, T, C), (b.d_ss, C, 1))
        _within("du", du, r["du"], 2.0 ** -20 * r["duabs"])
        _untouched("du", b.du_buf, (N, T, C), (b.d_ss, C, 1), b.doff)
    # pass 2 with the sums fed to the kernel
    M = float(N * T)
    m1, m2 = b.S1in / M, b.S2in / M
    gi = p["gamma"].double() * p["invstd"].double()
    dy = gi * (r["du"] - m1 - r["xh"] * m2)
    bound = gi.abs() * (r["duabs"] + m1.abs() + r["xh"].abs() * m2.abs())
    shape, strides = (N, T, C), (b.d_ss, C, 1)
    hi = _view(b.out(b.dst_buf), shape, strides)
    _untouched("dst", b.dst_buf, shape, strides, b.doff)
    if b.fmt == 0:
        _within("dy", hi, dy, 2.0 ** -20 * bound)
        if b.lo_buf is not None:
            _untouched("dst_lo", b.lo_buf, shape, strides, b.doff)
            d, lo = hi.contiguous(), _view(b.out(b.lo_buf), shape, strides).contiguous()
            rec = emul.core._tf32_trunc(d) + lo
            _within("trunc_tf32(dst) + dst_lo", rec, d.double(), 2.0 ** -21 * d.double().abs())
            assert torch.equal(lo, emul.core._residual(d)), "dst_lo != residual(dst)"
    elif b.fmt == 1:
        _within("dy (bf16)", hi, dy, _ulp(dy, 7) + 2.0 ** -20 * bound)
    else:
        _untouched("dst_lo", b.lo_buf, shape, strides, b.doff)
        # the kernel's power-of-two scale from its own pass-1 maxima, in fp32
        g32 = (p["gamma"] * p["invstd"]).abs()
        s1 = (b.S1in * (1.0 / M)).float().abs()
        s2 = (b.S2in * (1.0 / M)).float().abs()
        bnd = float((g32 * (b.amax[0] + s1 + b.amax[1] * s2)).max())
        s = emul.core.f16_grad_scale(bnd * 1.0001)
        assert b.scale_out.tolist() == [1.0 / s, s], (b.scale_out.tolist(), s)
        v = hi.double() + _view(b.out(b.lo_buf), shape, strides).double() / 2048.0
        assert float(v.abs().max()) <= 16384.0
        _within("dy (fp16 pair)", v, s * dy, s * bound * (2.0 ** -20 + 2.0 ** -21) + 2.0 ** -35)
    if b.db is not None:
        pr = b.prior["db"]
        _within("db", b.db, pr + dy.sum((0, 1)),
                2.0 ** -16 * bound.sum((0, 1)) + 2.0 ** -40 * pr.abs())


def _print_plans(name, p1, p2):
    print("%s: pass 1 %s, pass 2 %s" % (name, p1, p2))


def _assert_staged(p):
    assert p["path"] == 1, p
    # more than STAGES tiles in some block, here and on any device with up to MAX_SMS SMs
    assert p["items"] > STAGES * p["grid"] and p["items"] > STAGES * 2 * MAX_SMS, p


def _assert_grid_stride(b, p):
    """Register kernel whose threads loop: more runs than threads, here and for any SM count
    up to MAX_SMS (the grid cap is 8 x SMs blocks over the samples)."""
    assert p["path"] == 0, p
    assert p["items"] > p["grid"] * THREADS, p
    assert p["items"] > (8 * MAX_SMS + b.N) * THREADS, p


# id -> (Bwd arguments, expected path of pass 1, of pass 2)
CASES = {
    # staged kernels with the ring wrapping; T leaves the last tile of each sample partial
    "ring-C32": (dict(N=16, T=8001, C=32, padL=4, padR=5, pool_d=8), 1, 1),
    "ring-C64-3xtf32": (dict(N=16, T=4001, C=64, prec="3xtf32", padL=5, padR=5, pool_d=16), 1, 1),
    "ring-C128-bf16": (dict(N=16, T=2001, C=128, prec="bf16", padL=4, padR=5, pool_d=8), 1, 1),
    "ring-C256-3xf16": (dict(N=16, T=1001, C=256, prec="3xf16", padL=4, padR=5, pool_d=4), 1, 1),
    "ring-C512-bf16-a32": (dict(N=8, T=1001, C=512, prec="bf16-a32", padL=4, padR=5,
                                pool_d=2), 1, 1),
    "ring-C1024": (dict(N=4, T=1001, C=1024, padL=4, padR=5, pool_d=2), 1, 1),
    # the PASE+ last block: A = dsrc[C:] at row stride 2C, B = dsrc shifted by one step
    "lastblock-fp32": (dict(N=8, T=1001, C=512, interleaved=True), 1, 1),
    "lastblock-bf16-a32": (dict(N=8, T=1001, C=512, prec="bf16-a32", interleaved=True), 1, 1),
    "lastblock-3xf16": (dict(N=16, T=1001, C=256, prec="3xf16", interleaved=True), 1, 1),
    # reflect pads against 4- and 8-row tiles; row-by-row bulk copies (a_rs > C)
    "pad4-tile4-ars": (dict(N=4, T=1001, C=1024, padL=4, padR=5, a_rs=1024 + 32), 1, 1),
    "pad8-tile4-3xtf32": (dict(N=4, T=1002, C=1024, prec="3xtf32", padL=8, padR=8,
                               a_rs=1024 + 64), 1, 1),
    "pad8-tile8": (dict(N=8, T=1003, C=512, padL=8, padR=10), 1, 1),
    "pad5-tile8-3xf16": (dict(N=8, T=1001, C=512, prec="3xf16", padL=5, padR=4), 1, 1),
    "pad4-tile8-bf16": (dict(N=8, T=1005, C=512, prec="bf16", padL=4, padR=9), 1, 1),
    # pooling windows across tiles, wide concat pitch, T % pool_d != 0
    "pool160": (dict(N=8, T=8001, C=64, padL=9, padR=10, pool_d=160, p_rs=1920), 1, 1),
    "pool8-wide": (dict(N=16, T=2001, C=128, pool_d=8, p_rs=1920, a_rs=160), 1, 1),
    "pool2-wide-3xf16": (dict(N=8, T=1001, C=512, prec="3xf16", pool_d=2, p_rs=1920), 1, 1),
    # y pitch above T*C (sinc layer), offset dst at a pitch above T*C (taps - 1 zero rows)
    "pitches": (dict(N=16, T=2001, C=128, padL=4, padR=5, pool_d=8, y_ss=2004 * 128,
                     d_ss=2011 * 128, doff=10 * 128), 1, 1),
    "pitches-bf16": (dict(N=16, T=2001, C=128, prec="bf16", y_ss=2004 * 128, d_ss=2011 * 128,
                          doff=10 * 128), 1, 1),
    # register kernels, chosen by the input
    "reg-C48": (dict(N=3, T=1001, C=48, padL=4, padR=5, pool_d=8), 0, 0),
    "reg-C2048": (dict(N=2, T=301, C=2048, padL=5, padR=5, pool_d=4), 0, 0),
    "reg-bf16-yss4": (dict(N=4, T=1001, C=256, prec="bf16", padL=4, padR=5, pool_d=4,
                           y_ss=1001 * 256 + 4), 0, 0),
    "reg-dss4": (dict(N=16, T=1001, C=256, padL=4, padR=5, pool_d=4, d_ss=1001 * 256 + 4), 1, 0),
    "reg-dss4-3xtf32": (dict(N=16, T=1001, C=256, prec="3xtf32", d_ss=1001 * 256 + 4), 1, 0),
    # stored du: register kernels in both passes, every thread looping
    "reg-du-N32": (dict(N=32, T=8000, C=64, padL=4, padR=5, pool_d=16, du=True), 0, 0),
    # sinc layer (no bias gradient), eval mode, non-zero priors in every accumulator
    "nobias": (dict(N=16, T=2001, C=128, padL=4, padR=5, pool_d=8, dbias=False), 1, 1),
    "eval-3xtf32": (dict(N=16, T=1001, C=256, prec="3xtf32", pool_d=4, train=False), 1, 1),
    "eval-3xf16": (dict(N=16, T=1001, C=256, prec="3xf16", pool_d=4, train=False), 1, 1),
    "priors-3xf16": (dict(N=16, T=4001, C=64, prec="3xf16", padL=5, padR=5, pool_d=16,
                          priors=True), 1, 1),
    "priors-reg": (dict(N=3, T=1001, C=48, padL=4, padR=5, pool_d=8, priors=True), 0, 0),
    "priors-du": (dict(N=32, T=8000, C=64, pool_d=16, du=True, priors=True), 0, 0),
}


@pytest.mark.parametrize("case", list(CASES))
def test_bn_prelu_bwd_regimes(case):
    kw, path1, path2 = CASES[case]
    b = Bwd(seed=list(CASES).index(case), **kw)
    p1, p2 = b.plans()
    _print_plans(case, p1, p2)
    assert (p1["path"], p2["path"]) == (path1, path2), (p1, p2)
    for p, path in ((p1, path1), (p2, path2)):
        if path == 1:
            _assert_staged(p)
    if kw.get("du"):
        _assert_grid_stride(b, p1)
        _assert_grid_stride(b, p2)
    b.run()
    _check_bwd(b, _bwd_reference(b))


def test_decoder_bwd_register_grid_stride():
    """The waveform decoder's last transposed-conv layer at B=32: pass 1 stores du (register
    kernel, every thread looping) at the decoder's y / du pitch U*s*C, pass 2 reads it."""
    from pase_b200.minions import DecoderMinion
    from pase_b200.decoder import DecoderPlan
    m = DecoderMinion(256, 1, 0.0)
    layers = [(b.deconv.weight.shape[0], b.deconv.weight.shape[1], b.kwidth, b.stride, b.pad)
              for b in m.blocks[:m.n_deconv]]
    g = DecoderPlan(layers, 32, 200, torch.device("meta")).geoms[-1]
    C = g.Cout
    b = Bwd(N=32, T=g.L, C=C, y_ss=g.U * g.s * C, d_ss=g.U * g.s * C, doff=g.pad * C, du=True,
            seed=77)
    p1, p2 = b.plans()
    _print_plans("decoder", p1, p2)
    _assert_grid_stride(b, p1)
    _assert_grid_stride(b, p2)
    b.run()
    _check_bwd(b, _bwd_reference(b))


@pytest.mark.parametrize("prec", ["fp32", "3xf16"])
def test_staged_bwd_is_reproducible(prec):
    """Both staged passes twice at a ring-wrapping shape: dy equal in every bit, the fp64
    sums equal once rounded to fp32."""
    res = []
    for _ in range(2):
        b = Bwd(N=16, T=4001, C=64, prec=prec, padL=5, padR=5, pool_d=16, seed=5)
        p1, p2 = b.plans()
        _assert_staged(p1)
        _assert_staged(p2)
        b.run()
        res.append(b)
    b1, b2 = res
    assert torch.equal(b1.dst_buf, b2.dst_buf)
    if b1.lo_buf is not None:
        assert torch.equal(b1.lo_buf, b2.lo_buf)
    for k in ("S1", "S2", "dal", "db"):
        x, z = getattr(b1, k), getattr(b2, k)
        assert float((x - z).abs().max()) <= 1e-14 * float(x.abs().max())
        assert torch.equal(x.float(), z.float()), k
    if prec == "3xf16":
        assert torch.equal(b1.amax, b2.amax) and torch.equal(b1.scale_out, b2.scale_out)


# ---- forward: a = PReLU(y*scale + shift) into the next layer's padded operand + pooling ----
class Fwd(object):
    def __init__(self, N, T, C, prec="fp32", padL=0, padR=0, y_ss=None, d_rs=None, d_ss=None,
                 doff=0, pool_d=0, pool_T=None, p_rs=None, p_ss=None, p_off=0, priors=False,
                 seed=0):
        gen = torch.Generator(device="cuda").manual_seed(2000 + seed)
        self.N, self.T, self.C = N, T, C
        self.ybf, _, self.fmt, lo = PRECS[prec]
        self.p = _bn_params(C, gen)
        self.y_ss = y_ss if y_ss is not None else T * C
        self.y = _make_y(N, T, C, self.y_ss, self.ybf, self.p, gen)
        self.padL, self.padR = padL, padR
        self.Tp = T + padL + padR
        self.d_rs = d_rs if d_rs is not None else C
        self.d_ss = d_ss if d_ss is not None else self.Tp * self.d_rs
        self.doff = doff
        odt = FMT_DTYPE[self.fmt]
        n_out = doff + N * self.d_ss + 64
        self.dst_buf = _guarded(n_out, odt)
        self.lo_buf = _guarded(n_out, odt) if lo else None
        self.pool_d = pool_d
        self.pool_T = pool_T if pool_T is not None else (T // pool_d if pool_d else 0)
        if pool_d:
            self.p_rs = p_rs if p_rs is not None else C + 64
            self.p_ss = p_ss if p_ss is not None else (self.pool_T + 1) * self.p_rs
            self.Pbuf = _guarded(p_off + N * self.p_ss + self.p_rs, torch.float32)
            self.P = self.Pbuf[p_off:]
            self.pview = _view(self.P, (N, self.pool_T, C), (self.p_ss, self.p_rs, 1))
            self.prior = _randn(N * self.pool_T * C, gen).view(N, self.pool_T, C) if priors \
                else torch.zeros(N, self.pool_T, C, device="cuda")
            self.pview.copy_(self.prior)
            self.p_off = p_off
        else:
            self.P, self.p_rs, self.p_ss = None, 0, 0

    def run(self):
        p = self.p
        _lib.call("pase_bn_prelu_pad_fwd", self.y, self.ybf, self.y_ss, self.N, self.T, self.C,
                  p["scale"], p["shift"], p["alpha"], self.dst_buf[self.doff:],
                  None if self.lo_buf is None else self.lo_buf[self.doff:], self.fmt, self.d_ss,
                  self.d_rs, self.padL, self.padR, self.P, self.p_ss, self.p_rs, self.pool_d,
                  self.pool_T)
        torch.cuda.synchronize()

    def check(self):
        N, T, C, p = self.N, self.T, self.C, self.p
        y = _view(self.y, (N, T, C), (self.y_ss, C, 1)).double()
        u = y * p["scale"].double() + p["shift"].double()
        a = torch.where(u > 0, u, p["alpha"].double() * u)
        idx = (torch.arange(self.Tp, device="cuda") - self.padL).abs()
        idx = torch.where(idx >= T, 2 * (T - 1) - idx, idx)
        ref = a[:, idx]
        shape, strides = (N, self.Tp, C), (self.d_ss, self.d_rs, 1)
        hi = _view(self.dst_buf[self.doff:], shape, strides)
        _untouched("dst", self.dst_buf, shape, strides, self.doff)
        if self.fmt == 0:
            _within("a", hi, ref, 2 * _ulp(ref, 23))
            if self.lo_buf is not None:
                _untouched("dst_lo", self.lo_buf, shape, strides, self.doff)
                d = hi.contiguous()
                lo = _view(self.lo_buf[self.doff:], shape, strides).contiguous()
                rec = emul.core._tf32_trunc(d) + lo
                _within("trunc_tf32(dst) + dst_lo", rec, d.double(), 2.0 ** -21 * d.double().abs())
                assert torch.equal(lo, emul.core._residual(d)), "dst_lo != residual(dst)"
        elif self.fmt == 1:
            _within("a (bf16)", hi, ref, _ulp(ref, 7))
        else:
            _untouched("dst_lo", self.lo_buf, shape, strides, self.doff)
            v = hi.double() + _view(self.lo_buf[self.doff:], shape, strides).double() / 2048.0
            _within("a (fp16 pair)", v, ref, 2 * _ulp(ref, 23) + 2.0 ** -22 * ref.abs() + 2.0 ** -35)
        if self.P is None:
            return
        # window means of what the next layer reads: the bf16 operand as stored, else a itself
        L, d = self.pool_T * self.pool_d, self.pool_d
        seen = hi[:, self.padL:self.padL + L].double() if self.fmt == 1 else a[:, :L]
        mean = seen.reshape(N, self.pool_T, d, C).mean(2)
        mabs = seen.abs().reshape(N, self.pool_T, d, C).mean(2)
        ref_p = self.prior.double() + mean
        _within("pool", self.pview, ref_p, (d + 4) * U * mabs + U * ref_p.abs())
        _untouched("pool", self.Pbuf, (N, self.pool_T, C), (self.p_ss, self.p_rs, 1), self.p_off)


FWD_CASES = {
    "pool160-fp32": dict(N=8, T=8001, C=64, padL=9, padR=10, pool_d=160, p_rs=1920),
    "pool2-3xtf32": dict(N=4, T=1001, C=1024, prec="3xtf32", padL=4, padR=5, pool_d=2,
                         p_rs=1920, priors=True),
    "pool8-bf16": dict(N=8, T=1003, C=512, prec="bf16", padL=8, padR=10, pool_d=8, p_rs=1920),
    "pool8-3xf16": dict(N=8, T=2001, C=128, prec="3xf16", padL=5, padR=5, pool_d=8),
    "pitches-C48": dict(N=3, T=1001, C=48, padL=4, padR=5, pool_d=16, y_ss=1004 * 48,
                        d_rs=56, d_ss=1012 * 56, doff=56, priors=True),
    "nopool-bf16-yss4": dict(N=4, T=1001, C=256, prec="bf16", y_ss=1001 * 256 + 4, padL=5,
                             padR=5),
}


@pytest.mark.parametrize("case", list(FWD_CASES))
def test_bn_prelu_pad_fwd_regimes(case):
    f = Fwd(seed=list(FWD_CASES).index(case), **FWD_CASES[case])
    f.run()
    f.check()


# ---- the PASE+ step's own geometry: every block at N=32, T=32000 ----
def _pasep_plan(prec):
    from helpers import resolve_cfg
    from pase_b200 import wf_builder
    cfg = wf_builder(resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    return E.EncoderPlan(cfg, 32, 32000, torch.device("meta"), prec)


@pytest.mark.parametrize("prec", ["fp32", "3xtf32", "bf16", "3xf16"])
def test_pasep_step_geometry(prec):
    """Forward and both backward passes of every PASE+ block with the arguments the training
    step passes (encoder_forward / encoder_backward_steps), geometry from EncoderPlan."""
    plan = _pasep_plan(prec)
    G, N, Tq, Kc = plan.geoms, plan.N, plan.Tq, plan.Kc
    assert plan.rnn and plan.skips
    for l, g in enumerate(G):
        C, last = g.Cout, l == plan.nblk - 1
        pool = {} if last else dict(pool_d=plan.pool_d[l], pool_T=Tq, p_ss=Tq * Kc, p_rs=Kc,
                                    p_off=plan.col_off[l])
        if last:            # QRNN input operand xq[C:] at pitch (Tq + 1) C, no halo
            fwd = dict(d_ss=(Tq + 1) * C, d_rs=C, doff=C)
        else:
            nx = G[l + 1]
            fwd = dict(padL=nx.padL, padR=nx.padR, d_ss=nx.apad_floats, d_rs=C)
        f = Fwd(N, g.T_out, C, prec, y_ss=g.Ty * C, seed=l, **fwd, **pool)
        f.run()
        f.check()
        del f
        bprec = "bf16-a32" if (prec == "bf16" and last) else prec
        if last:
            src = dict(interleaved=True)
        else:
            src = dict(padL=nx.padL, padR=nx.padR, a_ss=nx.apad_floats, a_rs=C)
        doff = 0 if g.sinc else (g.taps - 1) * C
        d_ss = g.Ty * C if g.sinc else g.Pd * C
        b = Bwd(N, g.T_out, C, bprec, y_ss=g.Ty * C, d_ss=d_ss, doff=doff, dbias=not g.sinc,
                seed=100 + l, **src, **pool)
        p1, p2 = b.plans()
        _print_plans("%s block %d (C=%d T=%d)" % (prec, l, C, g.T_out), p1, p2)
        assert p1["path"] == 1 and p2["path"] == 1, (p1, p2)
        b.run()
        _check_bwd(b, _bwd_reference(b))
        del b
        torch.cuda.empty_cache()


# ---- operands the kernels cannot address are refused before any launch ----
def _base_args(name, N=2, T=64, C=64, padL=2, padR=2, pool_d=4):
    """Valid fp32 arguments of `name`, by parameter name."""
    dev = dict(device="cuda")
    Tp = T + padL + padR
    vec = lambda: torch.ones(C, **dev)
    f64 = lambda: torch.zeros(C, dtype=torch.float64, **dev)
    kw = dict(y=torch.zeros(N * T * C + 64, **dev), y_bf16=0, y_sample_stride=T * C, N=N, T=T,
              C=C, mean=vec(), invstd=vec(), gamma=vec(), scale=vec(), shift=vec(), alpha=vec(),
              srcA=torch.zeros(N * Tp * C + 64, **dev), a_bf16=0, a_sample_stride=Tp * C,
              a_row_stride=C, padL=padL, padR=padR, srcB=torch.zeros(N * T * C + 64, **dev),
              b_sample_stride=T * C, b_row_stride=C, b_shift=1,
              pool=torch.zeros(N * (T // pool_d) * C + 64, **dev),
              pool_sample_stride=(T // pool_d) * C, pool_row_stride=C, pool_d=pool_d,
              pool_T=T // pool_d, dst=torch.zeros(N * Tp * C + 64, **dev),
              dst_lo=torch.zeros(N * Tp * C + 64, **dev), dst_fmt=0,
              dst_sample_stride=(Tp if name == "pase_bn_prelu_pad_fwd" else T) * C,
              dst_row_stride=C, S1=f64(), S2=f64(), dalpha=f64(), amax=None,
              count=float(N * T), du=torch.zeros(N * T * C + 64, **dev), dbias_acc=f64(),
              scale_out=None)
    if name == "pase_bn_prelu_bwd_reduce":
        kw["dst"] = None               # sums only
    return kw


def _call(name, kw):
    params = [p for (_, _, p) in _lib.PROTOS[name][1] if p != "stream"]
    return _lib.call(name, *[kw[p] for p in params])


_BWD = ["pase_bn_prelu_bwd_reduce", "pase_bn_prelu_bwd_apply", "pase_bn_prelu_bwd_apply_src"]
_ALL = _BWD + ["pase_bn_prelu_pad_fwd"]
_SRC = ["pase_bn_prelu_bwd_reduce", "pase_bn_prelu_bwd_apply_src"]
_POOL = _SRC + ["pase_bn_prelu_pad_fwd"]
# (argument, entry points, bad value as a function of the valid arguments, message pattern)
_REJECT = [
    ("y", _ALL, lambda kw: kw["y"].data_ptr() + 4, r": y must be 16-byte aligned"),
    ("srcA", _SRC,
     lambda kw: kw["srcA"].data_ptr() + 8, r": srcA must be 16-byte aligned"),
    ("srcB", _SRC,
     lambda kw: kw["srcB"].data_ptr() + 4, r": srcB must be 16-byte aligned"),
    ("pool", _POOL, lambda kw: kw["pool"].data_ptr() + 12, r": pool must be 16-byte aligned"),
    ("dst", _ALL, lambda kw: kw["dst"].data_ptr() + 4, r": dst must be 16-byte aligned"),
    ("dst_lo", ["pase_bn_prelu_bwd_apply", "pase_bn_prelu_bwd_apply_src",
                "pase_bn_prelu_pad_fwd"],
     lambda kw: kw["dst_lo"].data_ptr() + 8, r": dst_lo must be 16-byte aligned"),
    ("du", ["pase_bn_prelu_bwd_apply"], lambda kw: kw["du"].data_ptr() + 4,
     r": du must be 16-byte aligned"),
    ("y_sample_stride", _ALL, lambda kw: kw["y_sample_stride"] + 2, r": y_sample_stride="),
    ("a_sample_stride", _SRC,
     lambda kw: kw["a_sample_stride"] - 1, r": a_sample_stride="),
    ("a_row_stride", _SRC,
     lambda kw: kw["C"] + 2, r": a_row_stride=66 must be a multiple of 4"),
    ("a_row_stride", _SRC,
     lambda kw: kw["C"] - 4, r": a_row_stride=60 < C=64"),
    ("b_sample_stride", _SRC,
     lambda kw: kw["b_sample_stride"] + 1, r": b_sample_stride="),
    ("b_row_stride", _SRC,
     lambda kw: kw["C"] + 2, r": b_row_stride=66 must be a multiple of 4"),
    ("b_row_stride", _SRC,
     lambda kw: kw["C"] - 8, r": b_row_stride=56 < C=64"),
    ("pool_sample_stride", _POOL, lambda kw: kw["pool_sample_stride"] + 2,
     r": pool_sample_stride="),
    ("pool_row_stride", _POOL, lambda kw: kw["C"] + 1, r": pool_row_stride="),
    ("pool_T", _POOL, lambda kw: kw["pool_T"] + 1, r": pool_T=17 x pool_d=4 exceeds T=64"),
    ("dst_sample_stride", _ALL, lambda kw: kw["dst_sample_stride"] + 2, r": dst_sample_stride="),
    ("dst_row_stride", ["pase_bn_prelu_pad_fwd"], lambda kw: kw["C"] + 2, r": dst_row_stride="),
]
_REJECT_IDS = []
for _arg, _fns, _bad, _pat in _REJECT:
    for _fn in _fns:
        _REJECT_IDS.append(pytest.param(_fn, _arg, _bad, _pat, id="%s-%s-%s" % (
            _fn[len("pase_bn_prelu_"):], _arg, "lt-C" if "<" in _pat else "bad")))


@pytest.mark.parametrize("fn,arg,bad,pattern", _REJECT_IDS)
def test_bn_prelu_rejects_unaddressable_operands(fn, arg, bad, pattern):
    kw = _base_args(fn)
    if fn == "pase_bn_prelu_bwd_reduce" and arg.startswith("dst"):
        kw["dst"] = kw["du"]                   # pass 1 storing du
    _call(fn, kw)                              # the valid call goes through
    torch.cuda.synchronize()
    kw[arg] = bad(kw)
    with pytest.raises(RuntimeError, match=fn + pattern):
        _call(fn, kw)


def test_bn_prelu_bf16_operands_need_8_byte_alignment():
    """16-bit operands are read in 8-byte quads: 8-byte alignment is enough, 4 is refused."""
    fn = "pase_bn_prelu_bwd_reduce"
    kw = _base_args(fn)
    y16 = torch.zeros(kw["y"].numel(), dtype=torch.bfloat16, device="cuda")
    kw.update(y=y16[4:], y_bf16=1, srcA=kw["srcA"].to(torch.bfloat16)[4:], a_bf16=1)
    p = _lib.bn_bwd_plan(1, *[kw[k] for k in (
        "y", "y_bf16", "y_sample_stride", "N", "T", "C", "srcA", "a_bf16", "a_sample_stride",
        "a_row_stride", "padL", "padR", "srcB", "b_sample_stride", "b_row_stride", "b_shift",
        "pool", "pool_sample_stride", "pool_row_stride", "pool_d", "pool_T")], None, None, 0, 0)
    assert p["path"] == 0, p                   # not 16-byte aligned: register kernels
    _call(fn, kw)
    torch.cuda.synchronize()
    kw["y"] = y16[2:]
    with pytest.raises(RuntimeError, match=fn + r": y must be 8-byte aligned"):
        _call(fn, kw)
