"""TEST-ONLY torch emulation of the entry points WaveFe.encode_long adds (include/pase_b200.h:
pase_out_bwd_gather_crop, pase_qrnn_scan_bwd_carry_var, pase_reflect_fold_wave_acc); the
windowed forward's entry points come from tests/emul_streams.py and the packed backward's from
tests/emul_packed_grad.py."""
import torch

import emul_input_grad
import emul_packed_grad
import emul_streams


def _rows(tab, n, width):
    return tab[:n * width].view(n, width).tolist()


def pase_out_bwd_gather_crop(dout, ld, col0, T, c0, cn, C, g):
    assert 0 <= c0 and c0 + cn <= T and col0 + cn <= ld
    v = torch.zeros(T, C)
    v[c0:c0 + cn] = dout[:C * ld].view(C, ld)[:, col0:col0 + cn].t()
    g[:T * C] = v.reshape(-1)


def pase_qrnn_scan_bwd_carry_var(Y, Cst, dh, lddh, dY, state, dstate, tab, nseg, H):
    rows = _rows(tab, nseg, 6)
    assert len({r[5] for r in rows}) == len(rows), "a slot twice in one launch"
    for row0, T, drow0, c0, cn, slot in rows:
        assert 0 <= c0 and c0 + cn <= T
        y = Y[row0 * 3 * H:(row0 + T) * 3 * H].view(T, 3 * H)
        z, f, o = torch.tanh(y[:, :H]), torch.sigmoid(y[:, H:2 * H]), torch.sigmoid(y[:, 2 * H:])
        c = Cst[row0 * H:(row0 + T) * H].view(T, H)
        out = torch.zeros(T + 1, 3 * H)
        carry = dstate[slot * H:(slot + 1) * H].clone()
        for t in range(c0 + cn - 1, c0 - 1, -1):
            g = dh[(row0 + t) * lddh:(row0 + t) * lddh + H]
            cm1 = c[t - 1] if t > c0 else state[slot * H:(slot + 1) * H]
            dc = g * o[t] + carry
            out[t, :H] = dc * f[t] * (1 - z[t] ** 2)
            out[t, H:2 * H] = dc * (z[t] - cm1) * f[t] * (1 - f[t])
            out[t, 2 * H:] = g * c[t] * o[t] * (1 - o[t])
            carry = dc * (1 - f[t])
        dY[drow0 * 3 * H:(drow0 + T + 1) * 3 * H] = out.reshape(-1)
        dstate[slot * H:(slot + 1) * H] = carry


def pase_reflect_fold_wave_acc(dpad, dx, x0, T, padL, padR, fold_l, fold_r):
    d = dpad[:T + padL + padR]
    v = d[padL:padL + T].clone()
    if fold_l:
        v[1:padL + 1] += d[:padL].flip(0)
    if fold_r:
        v[T - 1 - padR:T - 1] += d[T + padL:T + padL + padR].flip(0)
    dx[x0:x0 + T] += v


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        if hasattr(emul_streams, name):
            return emul_streams.call(name, *args)
        if hasattr(emul_packed_grad, name) or hasattr(emul_input_grad, name):
            return emul_packed_grad.call(name, *args)
        return emul_streams.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
