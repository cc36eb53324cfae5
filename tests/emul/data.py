"""The training-data entry points: batch assembly (pase_b200/csrc/batch.cu) with torch's CPU
fp32 operations, and the waveform distortions (pase_b200/csrc/distort.cu) in float64."""
import ctypes
import math

import numpy as np
import torch

BLK = 4096
FFT_N = 8192


def _row(buf, b, ld, n):
    flat = buf.reshape(-1)
    return flat[b * ld:b * ld + n]


# ---- batch assembly
def pase_chunk_gather(pcm, pcm_len, flt, flt_len, rows, B, nsrc, T, cchunk, out, plane):
    R = rows.reshape(B, nsrc, 6).tolist()
    flat = out.reshape(-1)
    for b in range(B):
        for s in range(nsrc):
            fmt, off, L, beg, scale, rbits = R[b][s]
            assert L >= 1 and (beg + T <= L or (beg == 0 and T - L < L))
            if fmt == 0:
                u = pcm[off:off + L].float() * (1.0 / 32768)
            else:
                u = flt[off:off + L]
            p = torch.arange(beg, beg + T)
            p = torch.where(p >= L, 2 * L - 2 - p, p)
            x = u[p]
            if scale:
                r = torch.from_numpy(np.array([rbits], np.int32).view(np.float32))
                x = x / torch.max(torch.abs(x)) * r
            flat[s * plane + b * T:s * plane + (b + 1) * T] = x
            if s == 0 and cchunk:
                flat[nsrc * plane + b * T:nsrc * plane + (b + 1) * T] = x


def pase_frames_gather(pool, pool_len, rows, B, F, n, out):
    for b, (off, frames, s) in enumerate(rows.reshape(B, 3).tolist()):
        assert s + n <= frames and off + F * frames <= pool_len
        X = pool[off:off + F * frames].view(F, frames)
        out[b].copy_(X[:, s:s + n])


# ---- distortions

def pase_fft_conv_workspace(njobs, T, Lmax, bytes_addr):
    nb = (T + Lmax - 1 + BLK - 1) // BLK
    pm = (Lmax + BLK - 1) // BLK
    ctypes.c_long.from_address(bytes_addr).value = (
        njobs * (nb + pm) * FFT_N * 8 + njobs * nb * 8 + njobs * T * 4)


def pase_fft_conv(x, ldx, bank, bank_len, jobs, njobs, T, Lmax, twiddle, ws, ws_bytes, out, ldo):
    J = jobs.reshape(njobs, 6).tolist()
    bk = bank.double().numpy()
    for b, (on, n, off, L, p, mode) in enumerate(J):
        if not on:
            continue
        assert 0 < n <= T and 0 < L <= Lmax and 0 <= p < L and off + L <= bank_len
        xr = _row(x, b, ldx, n).double().numpy()
        full = np.convolve(xr, bk[off:off + L])
        y = full[p:p + n].astype(np.float32)
        ex = float(np.dot(xr, xr))
        if mode == 2:
            res = y
        else:
            e = float(np.dot(full, full)) if mode == 1 else float(np.dot(y.astype(np.float64), y))
            if e > 0:
                res = np.float32(math.sqrt(ex / e)) * y
            else:
                res = y if mode == 1 else xr.astype(np.float32)
        _row(out, b, ldo, n).copy_(torch.from_numpy(np.ascontiguousarray(res, dtype=np.float32)))


def pase_segment_gather(pool, pool_len, jobs, njobs, T, out, ldo):
    for b, (on, off, avail) in enumerate(jobs.reshape(njobs, 3).tolist()):
        if not on:
            continue
        assert 0 <= avail <= T and off + avail <= pool_len
        r = torch.zeros(T, dtype=torch.float32)
        r[:avail] = pool[off:off + avail]
        _row(out, b, ldo, T).copy_(r)


def pase_noise_mix(x, ldx, seg, lds, jobs, snr_lin, njobs, T):
    for b, (on, shift, guard) in enumerate(jobs.reshape(njobs, 3).tolist()):
        if not on:
            continue
        xr = _row(x, b, ldx, T)
        n = torch.zeros(T, dtype=torch.float64)
        n[shift:] = _row(seg, b, lds, T - shift).double()
        xd = xr.double()
        ex, en = float(xd.dot(xd)), float(n.dot(n))
        if guard and not en > 0:
            continue
        K = math.sqrt(ex / (float(snr_lin[b]) * en)) if en > 0 else 1.0
        v = xd + K * n
        xr.copy_((math.sqrt(ex / (float(v.dot(v)) + 1e-14)) * v).float())


def pase_clip(x, ldx, jobs, cf, njobs, T):
    for b in range(njobs):
        if int(jobs[b]) == 0:
            continue
        xr = _row(x, b, ldx, T)
        lo, hi = float(cf[b]) * float(xr.min()), float(cf[b]) * float(xr.max())
        xr.copy_(torch.minimum(torch.maximum(xr, torch.tensor(lo, dtype=torch.float32)),
                               torch.tensor(hi, dtype=torch.float32)))


def pase_overlap_label(jobs, njobs, T, d, label, ldl):
    for b, (on, shift, _) in enumerate(jobs.reshape(njobs, 3).tolist()):
        m = torch.zeros(T, dtype=torch.float32)
        if on:
            m[shift:] = 1
        _row(label, b, ldl, T // d).copy_(m.view(-1, d).sum(1) / d)
