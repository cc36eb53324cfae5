"""The windowed entry points that StreamPool, and so FeatureStream, WaveFe.extract_long and
WaveFe.encode_long, launch: the stream ring gather, the QRNN scans that carry their state across
windows, and the placement / cropping of each window's output."""
import torch

from pase_b200.modules import select_output

from .core import _MODES, _rows


# ---- forward
def pase_stream_gather(staging, ring, ring_cap, wave, tab, nrow, max_len):
    for slot, head, nnew, so, rs, old, sl, wo in _rows(tab, nrow, 8):
        assert 0 <= nnew <= max_len and 0 <= sl <= max_len
        r = ring[slot * ring_cap:(slot + 1) * ring_cap]
        read = [(rs + i) % ring_cap for i in range(min(max(old, 0), sl))]
        write = [(head + i) % ring_cap for i in range(nnew)]
        assert not set(read) & set(write), "a row appends where its segment reads"
        seg = torch.empty(sl)
        if read:
            seg[:len(read)] = r[torch.tensor(read, dtype=torch.long)]
        if sl > len(read):
            a = len(read) - old                         # first staging sample of the segment
            seg[len(read):] = staging[so + a:so + a + sl - len(read)]
        wave[wo:wo + sl] = seg
        if write:
            r[torch.tensor(write, dtype=torch.long)] = staging[so:so + nnew]


def pase_qrnn_scan_fwd_carry_var(Y, h, ldh, Cst, state, tab, nseg, H):
    rows = _rows(tab, nseg, 4)
    assert len({r[2] for r in rows}) == len(rows), "a slot twice in one launch"
    for row0, T, slot, first in rows:
        st = state[slot * H:(slot + 1) * H]
        y = Y[row0 * 3 * H:(row0 + T) * 3 * H].view(T, 3 * H)
        z, f, o = torch.tanh(y[:, :H]), torch.sigmoid(y[:, H:2 * H]), torch.sigmoid(y[:, 2 * H:])
        c = torch.zeros(H) if first else st.clone()
        for t in range(T):
            c = f[t] * z[t] + (1 - f[t]) * c
            Cst[(row0 + t) * H:(row0 + t + 1) * H] = c
            h[(row0 + t) * ldh:(row0 + t) * ldh + H] = o[t] * c
        st[:] = c


def pase_out_place_var(y, scale, shift, out, tab, nseg, max_T, C):
    for row0, T, ocol, ldo, col0 in _rows(tab, nseg, 5):
        assert T <= max_T
        # one rounding of y*scale + shift, as the kernel's fmaf
        v = (y[row0 * C:(row0 + T) * C].view(T, C).double() * scale[:C].double()
             + shift[:C].double()).float()
        out[ocol * C:ocol * C + C * ldo].view(C, ldo)[:, col0:col0 + T] = v.t()


def pase_out_select(out, T, C, mode):
    o = out.view(-1)
    h = o[:C * T].view(1, C, T).clone()
    f = select_output(h.double(), _MODES[mode]).float()
    o[:f.numel()] = f.reshape(-1)


# ---- backward
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
