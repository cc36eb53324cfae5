"""The kernels at both ends of the encoder step against a float64 reference computed with torch
from the same fp32 inputs, in the regimes the training step runs them:
  the sinc layer:   pase_sinc_make, pase_sinc_grad;
  the QRNN:         pase_qrnn_scan_fwd, pase_qrnn_scan_bwd;
  the output layer: pase_out_affine_nct, pase_out_bwd_reduce, pase_out_bwd_apply,
                    pase_bn_finalize, pase_bn_eval_affine, and the pase_colsum /
                    pase_transpose_pad calls that feed the QRNN and output GEMMs.
Geometry (N = 32, T' = 25 / 100 / 200 / 300, H = 512, Kc = 1920, C = 256, the sinc fold of
each precision) comes from EncoderPlan for PASE+ at T = 4001 / 16000 / 32000 / 48000.

Memory the kernels must not read (slack rows and columns of their inputs, the taps of dWp
outside each polyphase row's window) holds a huge finite sentinel, so a stray read shows up as
a large error; memory they must not write (the dense-skip columns [H, Kc) of the QRNN output,
slack rows, the tail of every output buffer) is checked unchanged.

Bounds (u = 2^-24).  fp32 library functions as the CUDA C++ Programming Guide's table of
single-precision maximum ulp errors gives them (default, non-fast-math build): expf, tanhf,
sinf, cosf 2 ulp over the full range; division and square root correctly rounded.  One ulp of
x is at most 2u |x|, so each of these functions is off by at most 4u relative.
  QRNN forward: sigmoid = 1 / (1 + expf(-x)) is off by at most 6u relative, so 1 - f is off by
    at most 6u f + u |1 - f|.  Every step of c_t = f_t z_t + (1 - f_t) c_{t-1} adds at most
    kappa u (|f_t z_t| + m_{t-1}) to the error, where m_t = |f_t z_t| + (1 - f_t) m_{t-1} bounds
    |c_t| and everything the time-segmented kernels form on the way to it (segment products,
    the fold of earlier segments); the error carries as
      e_t = (1 - f_t) e_{t-1} + kappa u (|f_t z_t| + m_{t-1}),   kappa = 32
    (gate functions 11u on f z and 7u on (1 - f) c, up to 16 roundings of a segment product,
    the fold's fused multiply-add and the step's own rounding).  Cst within e_t, h within
    o_t e_t + kappa u o_t m_t.
  QRNN backward (fed the kernel's own fp32 Cst): the mirror form for dc_t = g_t o_t + carry,
      eps_t = (1 - f_{t+1}) eps_{t+1} + kappa u (|g_t o_t| + M_{t+1}),
      M_t = |g_t o_t| + (1 - f_{t+1}) M_{t+1};
    dz within eps_t f (1 - z^2) + kappa u M_t f, df within eps_t |z - c_{t-1}| f (1 - f) +
    kappa u M_t (|z| + |c_{t-1}|) f, do within kappa u |g c| o.
  sinc filters: the phase high * n (up to ~390 rad) is rounded to fp32 (u |high n|), sinf adds
    4u |sin|; a tap is within |A| / 2b (E_S + u |S|) + 4u |f|, with A = window / (n / 2),
    S = sin(high n) - sin(low n), b = high - low and E_S = u (|high n| |cos(high n)| +
    |low n| |cos(low n)|) + 4u (|sin(high n)| + |sin(low n)|) + u^2 ((high n)^2 + (low n)^2).
    The centre tap is exactly 1, taps outside each row's window exactly 0.
  sinc cut-off gradients: the fp32 fold sum of a tap pair's 2 fold terms within
    (2 fold - 1) u sum|terms|, then per tap |g| |A| times the errors of cos (phase rounding
    u |high n| |sin| + 4u |cos|) and of S, and 1u / 2u for the fp32 band in 1/b and 1/b^2;
    fp64 accumulation 2^-40 of the sum of magnitudes, the final fp32 rounding 1u.  The clamp
    gate and high are the fp32 evaluation of (min_low + |l|) + min_band + |b|; the float64
    part starts after that.
  output layer: fmaf(y, scale, shift) and a single product within 1 ulp; g_ntc exact; sums
    (S1, S2, colsum) within 2^-16 of the sum of the terms' magnitudes (the BatchNorm/PReLU
    convention); the applied gradient within 2^-20 |scale| (|g| + |S1/M| + |xhat| |S2/M|).
  bn_finalize: 1 fp32 ulp, plus the fp64 cancellation of q/M - m^2 carried to each output.
Each case prints its worst error as a fraction of its bound.  test_bounds_hold_for_emulation
runs the fp32 torch emulation (tests/emul/) through the same references and bounds on the
CPU, and shows that moving one element by twice its bound fails."""
import pytest
import torch

import emul
from pase_b200 import _lib
from pase_b200 import encoder as E

U = 2.0 ** -24
SENT = 2.0 ** 100          # huge finite sentinel in memory the kernels must not read
GUARD = 2.0 ** 100         # guard value in memory the kernels must not write
K_QRNN = 32.0
MIN_LOW = MIN_BAND = 50.0
SR = 16000.0
SINC_K = 251
gpu = pytest.mark.gpu


# ---- comparison helpers ----
def _within(what, got, ref, tol):
    """err <= tol everywhere; -> worst err / tol."""
    err = (got.double() - ref).abs()
    tol = torch.as_tensor(tol, dtype=torch.float64, device=err.device).expand_as(err)
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err - tol, torch.zeros_like(err)).reshape(-1)))
        raise AssertionError("%s: %d/%d out of bound; worst at flat %d: got %.9e ref %.9e "
                             "err %.3e tol %.3e" % (what, int(bad.sum()), bad.numel(), i,
                                                    float(got.reshape(-1)[i]),
                                                    float(ref.reshape(-1)[i]),
                                                    float(err.reshape(-1)[i]),
                                                    float(tol.reshape(-1)[i])))
    pos = tol > 0
    return float((err[pos] / tol[pos]).max()) if bool(pos.any()) else 0.0


def _untouched(what, buf, shape, strides, off=0):
    """Every element of buf outside the strided view still holds GUARD."""
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    torch.as_strided(keep, shape, strides, off).fill_(False)
    rest = buf[keep]
    assert torch.equal(rest, torch.full_like(rest, GUARD)), what + ": guard written"


def _ulp32(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 23)


def _report(name, ratios):
    print("%s: worst err / bound %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios)))


def _full(n, v, dev, dtype=torch.float32):
    return torch.full((int(n),), v, dtype=dtype, device=dev)


def _call(dev, name, *args):
    """The CUDA kernel on a CUDA device, the fp32 torch emulation on the CPU."""
    if torch.device(dev).type == "cuda":
        _lib.call(name, *args)
        torch.cuda.synchronize()
    else:
        emul.call(name, *args)


# ---- PASE+ geometry ----
def _pasep_plan(T, prec="fp32"):
    from helpers import resolve_cfg
    from pase_b200 import wf_builder
    cfg = wf_builder(resolve_cfg("cfg/frontend/PASE+.cfg")).cfg
    return E.EncoderPlan(cfg, 32, T, torch.device("meta"), prec)


_PLAN_T = (4001, 16000, 32000, 48000)


def test_pasep_geometry():
    """The frame counts and widths the cases below are named after."""
    tq = [_pasep_plan(T).Tq for T in _PLAN_T]
    assert tq == [25, 100, 200, 300], tq
    p = _pasep_plan(32000)
    assert (p.N, p.H, p.Kc, p.emb, p.rows) == (32, 512, 1920, 256, 6400)
    for prec, fold, K in (("fp32", 4, 256), ("3xtf32", 32, 288), ("bf16", 64, 320)):
        g = _pasep_plan(32000, prec).geoms[0]
        assert (g.sinc, g.k, g.fold, g.K, g.Cout) == (True, SINC_K, fold, K, 64)


# ================================ QRNN ================================
class Qrnn(object):
    """Operands of one forward + backward scan.  Channel c % 3: 0 moderate gates (randn),
    1 saturated (|pre-activation| ~ 20: 1 - f is exactly 0 or 1 in fp32), 2 long memory
    (f pre-activation ~ -8: c_t depends on every earlier segment)."""

    def __init__(self, N, T, H, ld=None, dev="cuda", seed=0):
        self.N, self.T, self.H, self.dev = N, T, H, dev
        self.ld = ld if ld is not None else H + 1408           # Kc - H of PASE+
        gen = torch.Generator(device=dev).manual_seed(3000 + seed)
        rn = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32)
        sign = lambda *s: torch.where(rn(*s) > 0, 1.0, -1.0)
        kind = torch.arange(H, device=dev) % 3
        y = rn(N, T, 3, H)
        sat = sign(N, T, 3, H) * (20.0 + 0.5 * rn(N, T, 3, H))
        y = torch.where(kind == 1, sat, y)
        longf = -8.0 + 0.1 * rn(N, T, H)
        y[:, :, 1] = torch.where(kind == 2, longf, y[:, :, 1])
        rows = N * T
        self.Y = _full(rows * 3 * H + 64, SENT, dev)
        self.Y[:rows * 3 * H] = y.reshape(-1)
        # a segment's worth of slack rows: a write past T lands on guards inside the buffer
        self.h = _full((rows + 16) * self.ld, GUARD, dev)
        self.Cst = _full((rows + 16) * H, GUARD, dev)
        self.dh = _full((rows + 2) * self.ld, SENT, dev)
        self.hview(self.dh).copy_(rn(N, T, H))
        self.dY = _full(rows * 3 * H + 64, GUARD, dev)

    def hview(self, buf):
        return torch.as_strided(buf, (self.N, self.T, self.H), (self.T * self.ld, self.ld, 1))

    def fwd(self):
        _call(self.dev, "pase_qrnn_scan_fwd", self.Y, self.h, self.ld, self.Cst, self.N,
              self.T, self.H)

    def bwd(self):
        _call(self.dev, "pase_qrnn_scan_bwd", self.Y, self.Cst, self.dh, self.ld, self.dY,
              self.N, self.T, self.H)


def _qrnn_gates(q):
    N, T, H = q.N, q.T, q.H
    y = q.Y[:N * T * 3 * H].view(N, T, 3, H).double()
    return torch.tanh(y[:, :, 0]), torch.sigmoid(y[:, :, 1]), torch.sigmoid(y[:, :, 2])


def qrnn_fwd_checks(q):
    """[(what, got, ref, tol)] of the forward scan."""
    N, T, H = q.N, q.T, q.H
    z, f, o = _qrnn_gates(q)
    c, e, m = (torch.zeros(N, H, dtype=torch.float64, device=z.device) for _ in range(3))
    C, Eb, Mb = (torch.empty(N, T, H, dtype=torch.float64, device=z.device) for _ in range(3))
    for t in range(T):
        fz, a = f[:, t] * z[:, t], 1.0 - f[:, t]
        e = a * e + K_QRNN * U * (fz.abs() + m)
        c = fz + a * c
        m = fz.abs() + a * m
        C[:, t], Eb[:, t], Mb[:, t] = c, e, m
    return [("Cst", q.Cst[:N * T * H].view(N, T, H), C, Eb),
            ("h", q.hview(q.h), o * C, o * Eb + K_QRNN * U * o * Mb)]


def qrnn_bwd_checks(q):
    """[(what, got, ref, tol)] of the backward scan, fed the fp32 Cst of the forward kernel."""
    N, T, H = q.N, q.T, q.H
    z, f, o = _qrnn_gates(q)
    cs = q.Cst[:N * T * H].view(N, T, H).double()
    cm = torch.cat([torch.zeros_like(cs[:, :1]), cs[:, :-1]], 1)
    g = q.hview(q.dh).double()
    DC, Eps, Mb = (torch.empty(N, T, H, dtype=torch.float64, device=z.device) for _ in range(3))
    carry, eps, M = (torch.zeros(N, H, dtype=torch.float64, device=z.device) for _ in range(3))
    a_next = torch.zeros_like(carry)
    for t in range(T - 1, -1, -1):
        go = g[:, t] * o[:, t]
        dc = go + carry
        eps = a_next * eps + K_QRNN * U * (go.abs() + M)
        M = go.abs() + a_next * M
        DC[:, t], Eps[:, t], Mb[:, t] = dc, eps, M
        a_next = 1.0 - f[:, t]
        carry = dc * a_next
    dY = q.dY[:N * T * 3 * H].view(N, T, 3, H)
    kz, kf = f * (1.0 - z * z), (z - cm) * f * (1.0 - f)
    return [("dz", dY[:, :, 0], DC * kz, Eps * kz + K_QRNN * U * Mb * f),
            ("df", dY[:, :, 1], DC * kf,
             Eps * kf.abs() + K_QRNN * U * Mb * (z.abs() + cm.abs()) * f),
            ("do", dY[:, :, 2], g * cs * o * (1.0 - o), K_QRNN * U * (g * cs).abs() * o)]


def _check_all(checks):
    return [(w, _within(w, got, ref, tol)) for (w, got, ref, tol) in checks]


def _qrnn_untouched(q):
    N, T, H = q.N, q.T, q.H
    _untouched("h", q.h, (N, T, H), (T * q.ld, q.ld, 1))
    _untouched("Cst", q.Cst, (N * T * H,), (1,))


_QRNN_T = [1, 15, 16, 17, 200, 255, 256, 257, 300, 383, 384, 385, 511, 512, 513, 515, 1000]


def _expected_width(T):
    nseg = -(-T // 16)
    return 16 if nseg <= 16 else 24 if nseg <= 24 else 32 if nseg <= 32 else 0


def _qrnn_case(q, name):
    width = _lib.qrnn_scan_plan(q.T)
    assert width == _expected_width(q.T), (q.T, width)
    outs = []
    for _ in range(2):                  # no atomics: two runs give equal bits
        q.h.fill_(GUARD)
        q.Cst.fill_(GUARD)
        q.dY.fill_(GUARD)
        q.fwd()
        q.bwd()
        outs.append((q.h.clone(), q.Cst.clone(), q.dY.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b), "run-to-run difference"
    _qrnn_untouched(q)
    _untouched("dY", q.dY, (q.N * q.T * 3 * q.H,), (1,))
    r = _check_all(qrnn_fwd_checks(q)) + _check_all(qrnn_bwd_checks(q))
    _report("%s (%s)" % (name, "segments/block %d" % width if width else "sequential"), r)


@gpu
@pytest.mark.parametrize("T", _QRNN_T)
@pytest.mark.parametrize("H", [512, 33, 100])
def test_qrnn_scan_regimes(H, T):
    _qrnn_case(Qrnn(2, T, H, seed=T + H), "qrnn H=%d T=%d" % (H, T))


@gpu
@pytest.mark.parametrize("T", _PLAN_T)
def test_qrnn_scan_pasep_step(T):
    """N = 32, H = 512 at the step's own pitch ldh = lddh = Kc: h lands in columns [0, H) of the
    concatenated operand whose columns [H, Kc) hold the pooled dense skips."""
    p = _pasep_plan(T)
    _qrnn_case(Qrnn(p.N, p.Tq, p.H, ld=p.Kc, seed=T), "qrnn PASE+ T=%d (T'=%d)" % (T, p.Tq))


# ================================ sinc ================================
def sinc_edges32(l, b):
    """low, high and the clamp gate as the kernel evaluates them, in fp32."""
    low = l.abs() + MIN_LOW
    h = (low + MIN_BAND) + b.abs()
    hi = torch.tensor(SR * 0.5, dtype=torch.float32, device=l.device)
    clamped = (h < MIN_LOW) | (h > hi)
    return low, torch.clamp(torch.clamp(h, min=MIN_LOW), max=hi), clamped


def _sinc_terms(low, high, n, win):
    """float64 per-tap quantities of taps 0 .. k/2-1 (C, k/2)."""
    lo, hi = low.double()[:, None], high.double()[:, None]
    nn, w = n.double()[None, :], win.double()[None, :]
    b = hi - lo
    A = w / (nn / 2)
    ph, pl = hi * nn, lo * nn
    sh, sl, ch, cl = torch.sin(ph), torch.sin(pl), torch.cos(ph), torch.cos(pl)
    S = sh - sl
    ES = U * (ph.abs() * ch.abs() + pl.abs() * cl.abs()) + 4 * U * (sh.abs() + sl.abs()) \
        + U * U * (ph * ph + pl * pl)
    Ech = U * ph.abs() * sh.abs() + 4 * U * ch.abs() + U * U * ph * ph
    Ecl = U * pl.abs() * sl.abs() + 4 * U * cl.abs() + U * U * pl * pl
    return dict(b=b, A=A, S=S, ES=ES, ch=ch, cl=cl, Ech=Ech, Ecl=Ecl, n=nn)


def sinc_filter_ref(l, b, n, win):
    """float64 filters (C, k) and their bound."""
    low, high, _ = sinc_edges32(l, b)
    s = _sinc_terms(low, high, n, win)
    left = s["S"] * s["A"] / (2 * s["b"])
    tl = s["A"].abs() / (2 * s["b"]) * (s["ES"] + U * s["S"].abs()) + 4 * U * left.abs()
    one = torch.ones_like(left[:, :1])
    return (torch.cat([left, one, left.flip(1)], 1),
            torch.cat([tl, torch.zeros_like(one), tl.flip(1)], 1))


class Sinc(object):
    def __init__(self, fold, Kv, cut, C=64, dev="cuda", seed=0):
        self.C, self.k, self.fold, self.Kv, self.dev = C, SINC_K, fold, Kv, dev
        gen = torch.Generator(device="cpu").manual_seed(4000 + seed)
        if cut == "mel":
            from pase_b200.frontend import _SincParams
            sp = _SincParams(C, SINC_K, sample_rate=int(SR))
            l, b = sp.low_hz_.detach().reshape(-1), sp.band_hz_.detach().reshape(-1)
        else:
            l = torch.rand(C, generator=gen) * 4000.0
            b = torch.rand(C, generator=gen) * 2000.0
            edge = [(-300.0, 200.0),        # low_hz_ < 0
                    (0.0, 300.0),           # low_hz_ = 0
                    (500.0, -400.0),        # band_hz_ < 0
                    (700.0, 0.0),           # band_hz_ = 0
                    (-0.0, -0.0),           # both -0
                    (3000.0, 9000.0),       # high above sr/2: clamped
                    (0.0, 7900.0),          # high = sr/2 exactly: not clamped
                    (7880.0, 10.0),         # narrow band (60 Hz) up to 10 Hz below sr/2
                    (7890.0, -9.0),         # narrow band (59 Hz) up to 1 Hz below sr/2
                    (7949.0, 1.5)]          # high clamped to sr/2, 1 Hz above low
            for i, (lv, bv) in enumerate(edge):
                l[i], b[i] = lv, bv
        self.l, self.b = l.to(dev), b.to(dev)
        self.n, self.win = E.sinc_constants(SINC_K, SR, dev)
        self.filt = _full(C * SINC_K + 64, GUARD, dev)
        self.Wp = _full(fold * C * Kv + 64, GUARD, dev)
        # dWp: randn inside each row's window [p, p+k), the sentinel outside
        d = torch.randn(fold, C, Kv, generator=gen).to(dev)
        kk = torch.arange(Kv, device=dev)
        p = torch.arange(fold, device=dev)[:, None]
        inside = ((kk[None, :] >= p) & (kk[None, :] < p + SINC_K))[:, None, :]
        self.dWp = _full(fold * C * Kv + 64, SENT, dev)
        self.dWp[:fold * C * Kv] = torch.where(inside, d, torch.full_like(d, SENT)).reshape(-1)
        self.dlow = _full(C + 64, GUARD, dev)
        self.dband = _full(C + 64, GUARD, dev)

    def make(self):
        _call(self.dev, "pase_sinc_make", self.l, self.b, self.n, self.win, self.filt, self.Wp,
              self.C, self.k, self.fold, self.Kv, MIN_LOW, MIN_BAND, SR)

    def grad(self):
        _call(self.dev, "pase_sinc_grad", self.dWp, self.l, self.b, self.n, self.win, self.dlow,
              self.dband, self.C, self.k, self.fold, self.Kv, MIN_LOW, MIN_BAND, SR)


def sinc_make_checks(s):
    C, k, fold, Kv = s.C, s.k, s.fold, s.Kv
    ref, tol = sinc_filter_ref(s.l, s.b, s.n, s.win)
    filt = s.filt[:C * k].view(C, k)
    _untouched("filt", s.filt, (C * k,), (1,))
    assert bool((s.Wp[fold * C * Kv:] == GUARD).all()), "Wp: guard written"
    W = s.Wp[:fold * C * Kv].view(fold, C, Kv)
    for p in range(fold):          # row p is the filter shifted by p, exact zeros elsewhere
        assert torch.equal(W[p, :, p:p + k], filt), "Wp row %d != filt" % p
        assert bool((W[p, :, :p] == 0).all()) and bool((W[p, :, p + k:] == 0).all()), \
            "Wp row %d: taps outside [p, p+k) not zero" % p
    return [("filt", filt, ref, tol)]


def sinc_grad_ref(s):
    """float64 autograd of sum_p sum_j dWp[p, j+p] f_j (fp32 gate and high), and the bound."""
    C, k, fold = s.C, s.k, s.fold
    low, high, clamped = sinc_edges32(s.l, s.b)
    W = s.dWp[:fold * C * s.Kv].view(fold, C, s.Kv)
    G = sum(W[p, :, p:p + k].double() for p in range(fold))
    Gabs = sum(W[p, :, p:p + k].double().abs() for p in range(fold))
    lo = low.double().requires_grad_(True)
    hi = high.double().requires_grad_(True)
    with torch.enable_grad():
        nn, w = s.n.double()[None, :], s.win.double()[None, :]
        left = (torch.sin(hi[:, None] * nn) - torch.sin(lo[:, None] * nn)) / (nn / 2) * w \
            / (2 * (hi - lo)[:, None])
        f = torch.cat([left, torch.ones_like(left[:, :1]), left.flip(1)], 1)
        dlo, dhi = torch.autograd.grad((G * f).sum(), [lo, hi])
    open_ = (~clamped).double()
    dlow = (dlo + open_ * dhi) * torch.sign(s.l.double())
    dband = open_ * dhi * torch.sign(s.b.double())
    # bound, per tap pair i < k/2
    half = k // 2
    t = _sinc_terms(low, high, s.n, s.win)
    g = (G[:, :half] + G[:, k - half:].flip(1)).abs()
    gam = (2 * fold - 1) * U * (Gabs[:, :half] + Gabs[:, k - half:].flip(1))
    b, A, S, n = t["b"], t["A"].abs(), t["S"].abs(), t["n"].abs()
    th = (n * t["ch"].abs() / (2 * b) + S / (2 * b * b))
    tl = (n * t["cl"].abs() / (2 * b) + S / (2 * b * b))
    eh = gam * A * th + g * A * (n * t["Ech"] / (2 * b) + t["ES"] / (2 * b * b)
                                 + U * n * t["ch"].abs() / (2 * b) + 2 * U * S / (2 * b * b))
    el = gam * A * tl + g * A * (n * t["Ecl"] / (2 * b) + t["ES"] / (2 * b * b)
                                 + U * n * t["cl"].abs() / (2 * b) + 2 * U * S / (2 * b * b))
    mag = 2.0 ** -40 * (g * A * (th + tl)).sum(1)
    EH, EL = eh.sum(1) + mag, el.sum(1) + mag
    return dlow, dband, EL + open_ * EH + U * dlow.abs(), open_ * EH + U * dband.abs()


def sinc_grad_checks(s):
    C = s.C
    dlow, dband, tl, tb = sinc_grad_ref(s)
    _untouched("dlow", s.dlow, (C,), (1,))
    _untouched("dband", s.dband, (C,), (1,))
    return [("dlow", s.dlow[:C], dlow, tl), ("dband", s.dband[:C], dband, tb)]


_SINC = [("fp32", 4), ("3xtf32", 32), ("bf16", 64)]


@gpu
@pytest.mark.parametrize("cut", ["mel", "edges"])
@pytest.mark.parametrize("prec,fold", _SINC)
def test_sinc_make_and_grad(prec, fold, cut):
    g = _pasep_plan(32000, prec).geoms[0]
    assert g.fold == fold
    s = Sinc(fold, g.K, cut, C=g.Cout, seed=fold)
    low, high, clamped = sinc_edges32(s.l, s.b)
    if cut == "mel":      # the top channel's high is sr/2: on the clamp gate's boundary
        assert float(high[-1]) == SR / 2 and not bool(clamped[-1])
    else:
        assert clamped.tolist()[5:10] == [True, False, False, False, True]
        assert float(high[6]) == SR / 2
    s.make()
    r = _check_all(sinc_make_checks(s))
    s.grad()
    r += _check_all(sinc_grad_checks(s))
    dlow, dband = s.dlow[:s.C].clone(), s.dband[:s.C].clone()
    s.grad()
    assert torch.equal(dlow, s.dlow[:s.C]) and torch.equal(dband, s.dband[:s.C])
    _report("sinc fold %d K %d %s" % (fold, g.K, cut), r)


# ============================ output layer ============================
class Out(object):
    def __init__(self, N, T, C, dev="cuda", seed=0):
        self.N, self.T, self.C, self.dev = N, T, C, dev
        gen = torch.Generator(device=dev).manual_seed(5000 + seed)
        rn = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32)
        n = N * T * C
        self.y = _full(n + 64, SENT, dev)
        self.y[:n] = (rn(N, T, C) * 2.0 + rn(C)).reshape(-1)
        self.scale, self.shift = rn(C), rn(C)
        self.mean, self.invstd = rn(C) * 0.5, rn(C).abs() + 0.5
        self.dout = _full(n + 64, SENT, dev)
        self.dout[:n] = rn(n)
        self.dout_ntc = _full(n + 64, SENT, dev)
        self.dout_ntc[:n] = rn(n)
        self.prior = [rn(C).double() * 10, rn(C).double() * 10]


def out_affine_checks(o, ntc):
    N, T, C = o.N, o.T, o.C
    n = N * T * C
    out = _full(n + 64, GUARD, o.dev)
    out_ntc = _full(n + 64, GUARD, o.dev) if ntc else None
    _call(o.dev, "pase_out_affine_nct", o.y, o.scale, o.shift, out, out_ntc, N, T, C)
    ref = o.y[:n].view(N, T, C).double() * o.scale.double() + o.shift.double()
    _untouched("out", out, (n,), (1,))
    got = out[:n].view(N, C, T).permute(0, 2, 1)
    checks = [("out", got, ref, _ulp32(ref))]
    if ntc:
        _untouched("out_ntc", out_ntc, (n,), (1,))
        assert torch.equal(out_ntc[:n].view(N, T, C), got), "out_ntc != out^T"
    return checks


def out_bwd_checks(o, use_dout, use_ntc, use_stats):
    """pase_out_bwd_reduce, then pase_out_bwd_apply in place on its g."""
    N, T, C = o.N, o.T, o.C
    n = N * T * C
    g = _full(n + 64, GUARD, o.dev)
    S1, S2 = o.prior[0].clone(), o.prior[1].clone()
    dout = o.dout if use_dout else None
    dntc = o.dout_ntc if use_ntc else None
    _call(o.dev, "pase_out_bwd_reduce", dout, dntc, o.y, o.mean, o.invstd, N, T, C, g, S1, S2)
    _untouched("g_ntc", g, (n,), (1,))
    ref = torch.zeros(N, T, C, dtype=torch.float32, device=g.device)
    if use_dout:
        ref = ref + o.dout[:n].view(N, C, T).permute(0, 2, 1)
    if use_ntc:
        ref = ref + o.dout_ntc[:n].view(N, T, C)
    assert torch.equal(g[:n].view(N, T, C), ref), "g_ntc not exact"
    g64 = ref.double()
    xh = (o.y[:n].view(N, T, C).double() - o.mean.double()) * o.invstd.double()
    s1, s2 = g64.sum((0, 1)), (g64 * xh).sum((0, 1))
    checks = [("S1", S1, o.prior[0] + s1, 2.0 ** -16 * g64.abs().sum((0, 1))
               + 2.0 ** -40 * o.prior[0].abs()),
              ("S2", S2, o.prior[1] + s2, 2.0 ** -16 * (g64 * xh).abs().sum((0, 1))
               + 2.0 ** -40 * o.prior[1].abs())]
    # apply with the sums the kernel accumulated
    M = float(N * T)
    _call(o.dev, "pase_out_bwd_apply", g, o.y, o.mean, o.invstd, o.scale, S1, S2, M, use_stats,
          N * T, C)
    _untouched("dy", g, (n,), (1,))
    sc = o.scale.double()
    if use_stats:
        m1, m2 = S1 / M, S2 / M
        dy = sc * (g64 - m1 - xh * m2)
        tol = 2.0 ** -20 * sc.abs() * (g64.abs() + m1.abs() + xh.abs() * m2.abs())
    else:
        dy = sc * g64
        tol = _ulp32(dy)
    checks.append(("dy", g[:n].view(N, T, C), dy, tol))
    return checks


_OUT_T = {25: 4001, 200: 32000, 300: 48000}     # T' of PASE+ -> T


@gpu
@pytest.mark.parametrize("ntc", [False, True])
@pytest.mark.parametrize("T", list(_OUT_T))
def test_out_affine_nct(T, ntc):
    p = _pasep_plan(_OUT_T[T])
    assert p.Tq == T
    o = Out(p.N, T, p.emb, seed=T)
    _report("out_affine N=%d T=%d C=%d ntc=%d" % (p.N, T, p.emb, ntc),
            _check_all(out_affine_checks(o, ntc)))


@gpu
@pytest.mark.parametrize("use_stats", [1, 0])
@pytest.mark.parametrize("grads", ["dout", "dout_ntc", "both"])
@pytest.mark.parametrize("T", list(_OUT_T))
def test_out_bwd(T, grads, use_stats):
    o = Out(32, T, 256, seed=T + 7)
    ud, un = grads in ("dout", "both"), grads in ("dout_ntc", "both")
    _report("out_bwd N=32 T=%d C=256 %s use_stats=%d" % (T, grads, use_stats),
            _check_all(out_bwd_checks(o, ud, un, use_stats)))


# ---- BatchNorm finalisation at the step's counts ----
def bn_finalize_checks(C, fold, count, dev="cuda", running=True, seed=0):
    gen = torch.Generator(device=dev).manual_seed(6000 + seed)
    rn = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float64)
    mu = rn(C) * 2.0
    sd = rn(C).abs() + 0.1
    mu[0], sd[0] = 300.0, 0.3                       # |mean| >> std
    mu[1], sd[1] = -4000.0, 2.0
    parts = torch.rand(fold, C, generator=gen, device=dev, dtype=torch.float64) + 0.5
    parts = parts / parts.sum(0)
    cs = (parts * (count * mu)).reshape(-1)
    cq = (parts * (count * (sd * sd + mu * mu))).reshape(-1)
    gamma, beta = rn(C).float(), rn(C).float()
    rm0, rv0 = rn(C).float(), rn(C).abs().float() + 0.5
    rm, rv = _full(C + 64, GUARD, dev), _full(C + 64, GUARD, dev)
    rm[:C], rv[:C] = rm0, rv0
    outs = [_full(C + 64, GUARD, dev) for _ in range(4)]
    mom, eps = 0.1, 1e-5
    eps32 = torch.tensor(eps, dtype=torch.float32).item()     # the kernel's float eps
    _call(dev, "pase_bn_finalize", cs, cq, C, fold, float(count), gamma, beta,
          rm if running else None, rv if running else None, mom, eps, *outs)
    s = sum(cs.view(fold, C)[p] for p in range(fold))
    q = sum(cq.view(fold, C)[p] for p in range(fold))
    m = s / count
    var = q / count - m * m
    dvar = 8 * 2.0 ** -53 * (q / count + m * m)    # fp64 error of q/M - m^2
    rel = dvar / var
    is_ = 1.0 / torch.sqrt(var + eps32)
    g, b = gamma.double(), beta.double()
    ref = [m, is_, g * is_, b - m * g * is_]
    slack = [torch.zeros_like(m), 0.5 * rel * is_, 0.5 * rel * (g * is_).abs(),
             (0.5 * rel + 2.0 ** -50) * (m * g * is_).abs()]
    for buf in outs:
        _untouched("bn output", buf, (C,), (1,))
    checks = [(w, buf[:C], r, _ulp32(r) + sl) for w, buf, r, sl in
              zip(("mean", "invstd", "scale", "shift"), outs, ref, slack)]
    if running:
        _untouched("running_mean", rm, (C,), (1,))
        _untouched("running_var", rv, (C,), (1,))
        unb = var * count / (count - 1)
        m32 = torch.tensor(mom, dtype=torch.float32).item()
        rm_ref = (1 - m32) * rm0.double() + m32 * m
        rv_ref = (1 - m32) * rv0.double() + m32 * unb
        # + whether the momentum is taken as float (the C ABI) or as double
        dm = abs(mom - m32)
        checks += [("running_mean", rm[:C], rm_ref,
                    _ulp32(rm_ref) + 2.0 ** -50 * m.abs() + dm * (rm0.double() - m).abs()),
                   ("running_var", rv[:C], rv_ref,
                    _ulp32(rv_ref) + m32 * rel * unb + dm * (rv0.double() - unb).abs())]
    return checks


def _bn_cases():
    p = _pasep_plan(32000)
    cases = {"out-C256-fold1": (p.emb, 1, p.rows)}
    for prec in ("fp32", "3xtf32", "bf16"):
        g = _pasep_plan(32000, prec).geoms[0]
        cases["sinc-fold%d" % g.fold] = (g.Cout, g.fold, p.N * g.T_out)
    g = p.geoms[-1]
    cases["block7-C512-fold1"] = (g.Cout, 1, p.N * g.T_out)
    return cases


@gpu
@pytest.mark.parametrize("running", [True, False])
@pytest.mark.parametrize("case", ["out-C256-fold1", "sinc-fold4", "sinc-fold32", "sinc-fold64",
                                  "block7-C512-fold1"])
def test_bn_finalize(case, running):
    C, fold, count = _bn_cases()[case]
    _report("bn_finalize %s count %d" % (case, count),
            _check_all(bn_finalize_checks(C, fold, count, running=running, seed=fold)))


@gpu
def test_bn_eval_affine():
    C, dev = 256, "cuda"
    gen = torch.Generator(device=dev).manual_seed(6100)
    rn = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32)
    rm, rv, gamma, beta = rn(C) * 100, rn(C).abs() * 1e-3 + 1e-6, rn(C), rn(C)
    for gb in ((gamma, beta), (None, None)):
        outs = [_full(C + 64, GUARD, dev) for _ in range(4)]
        _call(dev, "pase_bn_eval_affine", rm, rv, gb[0], gb[1], C, 1e-5, *outs)
        is_ = 1.0 / torch.sqrt(rv.double() + torch.tensor(1e-5, dtype=torch.float32).item())
        g = gb[0].double() if gb[0] is not None else torch.ones_like(is_)
        b = gb[1].double() if gb[1] is not None else torch.zeros_like(is_)
        ref = [rm.double(), is_, g * is_, b - rm.double() * g * is_]
        for w, buf, r in zip(("mean", "invstd", "scale", "shift"), outs, ref):
            _untouched(w, buf, (C,), (1,))
            _within(w, buf[:C], r, _ulp32(r) * (0 if w == "mean" else 1))


# ---- column sums and transposes feeding the QRNN and output GEMMs ----
def colsum_checks(rows, C, ld, dev="cuda", seed=0):
    gen = torch.Generator(device=dev).manual_seed(7000 + seed)
    X = _full(rows * ld + 64, SENT, dev)
    xv = torch.as_strided(X, (rows, C), (ld, 1))
    xv.copy_(torch.randn(rows, C, generator=gen, device=dev) * 3 + 1)
    prior = torch.randn(C, generator=gen, device=dev, dtype=torch.float64)
    acc = _full(C + 64, GUARD, dev, torch.float64)
    acc[:C] = prior
    _call(dev, "pase_colsum", X, ld, rows, C, acc)
    assert bool((acc[C:] == GUARD).all()), "colsum: guard written"
    x64 = xv.double()
    return [("colsum", acc[:C], prior + x64.sum(0),
             2.0 ** -16 * x64.abs().sum(0) + 2.0 ** -40 * prior.abs())]


@gpu
@pytest.mark.parametrize("rows,C,ld", [(6400, 1536, 1536),      # the QRNN bias, T = 32000
                                       (6400, 256, 256),        # the output bias
                                       (300, 4133, 4144),       # across a 4096-column panel
                                       (7, 8193, 8200)])        # three panels, few rows
def test_colsum(rows, C, ld):
    _report("colsum %dx%d" % (rows, C), _check_all(colsum_checks(rows, C, ld, seed=C)))


def transpose_pad_check(rows, cols, lds, ldd, dev="cuda", seed=0):
    gen = torch.Generator(device=dev).manual_seed(7100 + seed)
    src = _full(rows * lds + 64, SENT, dev)
    sv = torch.as_strided(src, (rows, cols), (lds, 1))
    sv.copy_(torch.randn(rows, cols, generator=gen, device=dev))
    dst = _full(cols * ldd + 64, GUARD, dev)
    _call(dev, "pase_transpose_pad", src, lds, dst, ldd, rows, cols)
    dv = dst[:cols * ldd].view(cols, ldd)
    assert torch.equal(dv[:, :rows], sv.t()), "transpose not exact"
    assert bool((dv[:, rows:] == 0).all()), "padding not zero"
    assert bool((dst[cols * ldd:] == GUARD).all()), "transpose_pad: guard written"


@gpu
@pytest.mark.parametrize("rows,cols,lds,ldd", [(256, 1920, 1920, 256),     # Wcat -> WcatT
                                               (1536, 1024, 1024, 1536),   # Wq -> WqT
                                               (256, 1920, 1928, 300),
                                               (1536, 1024, 1100, 1571)])
def test_transpose_pad(rows, cols, lds, ldd):
    transpose_pad_check(rows, cols, lds, ldd, seed=rows + ldd)


# ---- refusals ----
@gpu
@pytest.mark.parametrize("arg,bad,pattern", [
    ("N", 0, r"N=0 T=5 C=8"), ("T", -1, r"N=2 T=-1 C=8"), ("C", 0, r"N=2 T=5 C=0"),
    ("y", None, r"null pointer")])
def test_out_bwd_reduce_refuses(arg, bad, pattern):
    dev = dict(device="cuda")
    kw = dict(dout=torch.zeros(80, **dev), dout_ntc=None, y=torch.zeros(80, **dev),
              mean=torch.zeros(8, **dev), invstd=torch.ones(8, **dev), N=2, T=5, C=8,
              g_ntc=torch.zeros(80, **dev), S1=torch.zeros(8, dtype=torch.float64, **dev),
              S2=torch.zeros(8, dtype=torch.float64, **dev))
    names = [p for (_, _, p) in _lib.PROTOS["pase_out_bwd_reduce"][1] if p != "stream"]
    _lib.call("pase_out_bwd_reduce", *[kw[p] for p in names])
    torch.cuda.synchronize()
    kw[arg] = bad
    with pytest.raises(RuntimeError, match="pase_out_bwd_reduce: " + pattern):
        _lib.call("pase_out_bwd_reduce", *[kw[p] for p in names])


@gpu
@pytest.mark.parametrize("fn,arg,bad,pattern", [
    ("fwd", "ldh", 7, r"ldh=7 < H=8"), ("bwd", "lddh", 4, r"lddh=4 < H=8"),
    ("fwd", "Y", None, r"null pointer"), ("fwd", "h", None, r"null pointer"),
    ("fwd", "Cst", None, r"null pointer"), ("bwd", "dh", None, r"null pointer"),
    ("bwd", "dY", None, r"null pointer"), ("bwd", "Cst", None, r"null pointer"),
    ("fwd", "T", 0, r"N=2 T=0 H=8"), ("bwd", "H", 0, r"N=2 T=5 H=0")])
def test_qrnn_scan_refuses(fn, arg, bad, pattern):
    dev = dict(device="cuda")
    N, T, H = 2, 5, 8
    kw = dict(Y=torch.zeros(N * T * 3 * H, **dev), h=torch.zeros(N * T * H, **dev), ldh=H,
              Cst=torch.zeros(N * T * H, **dev), dh=torch.zeros(N * T * H, **dev), lddh=H,
              dY=torch.zeros(N * T * 3 * H, **dev), N=N, T=T, H=H)
    name = "pase_qrnn_scan_" + fn
    names = [p for (_, _, p) in _lib.PROTOS[name][1] if p != "stream"]
    _lib.call(name, *[kw[p] for p in names])
    torch.cuda.synchronize()
    kw[arg] = bad
    with pytest.raises(RuntimeError, match=name + ": " + pattern):
        _lib.call(name, *[kw[p] for p in names])


# ---- the bounds are met by the fp32 emulation, and are not vacuous ----
def _emulated_checks():
    dev = "cpu"
    out = []
    for T, H in ((40, 33), (17, 6)):
        q = Qrnn(2, T, H, ld=H + 5, dev=dev, seed=T)
        q.fwd()
        q.bwd()
        _qrnn_untouched(q)
        out += [("qrnn T=%d " % T + w, g, r, t) for (w, g, r, t) in
                qrnn_fwd_checks(q) + qrnn_bwd_checks(q)]
    for cut in ("mel", "edges"):
        s = Sinc(4, 256, cut, C=16, dev=dev, seed=1)
        s.make()
        s.grad()
        out += [("sinc %s " % cut + w, g, r, t) for (w, g, r, t) in
                sinc_make_checks(s) + sinc_grad_checks(s)]
    o = Out(2, 37, 40, dev=dev, seed=1)
    out += out_affine_checks(o, True) + out_bwd_checks(o, True, True, 1) \
        + out_bwd_checks(o, True, False, 0)
    out += bn_finalize_checks(48, 4, 4000.0, dev=dev)
    out += colsum_checks(50, 70, 75, dev=dev)
    transpose_pad_check(37, 21, 23, 40, dev=dev)
    return out


def test_bounds_hold_for_emulation():
    checks = _emulated_checks()
    worst = _check_all(checks)
    _report("emulation", worst)
    tested = 0
    for w, got, ref, tol in checks:
        tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(got).reshape(-1)
        if not bool((tol > 0).any()):
            continue
        i = int(torch.argmax(tol))         # the loosest element of the check
        bumped = got.double().reshape(-1).clone()
        bumped[i] += 2 * tol[i]
        with pytest.raises(AssertionError, match="out of bound"):
            _within(w, bumped.view(got.shape), ref, tol.view(got.shape))
        tested += 1
    assert tested >= 20, tested
