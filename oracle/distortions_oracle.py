"""float64 numpy/scipy restatement of the six PASE+ waveform distortions the product runs on
the device (pase_b200/distortions.py), for one sample and an explicit plan.  Written from the
reference's documented behaviour (pase/transforms.py Reverb, SimpleAdditiveShift,
SimpleAdditive, Clipping, BandDrop, Downsample); the product never imports it.

banks: dict with raw float64 arrays as read from disk --
  'irs' (list), 'overlap' (list of noise wavs), 'noise' (list), 'bandrop' (list),
  'downsample' (list).
plan: the per-sample dict of DistortionPlan.samples[b].
"""
import numpy as np
from scipy import signal

MAX_REVERB_LEN = 24000


def _shift_left(full, p, n):
    """full[p : p + n] (the reference's shift(xs, -p) followed by the trim)."""
    return full[p:p + n]


def reverb(x, ir):
    h = np.asarray(ir, dtype=np.float64)[:MAX_REVERB_LEN]
    if np.max(h) > 0:
        h = h / abs(np.max(h))
    p = int(np.argmax(np.abs(h)))
    full = signal.convolve(x, h, mode="full")
    ex, er = float(np.dot(x, x)), float(np.dot(full, full))
    g = np.sqrt(ex / er) if er > 0 else 1.0
    return g * _shift_left(full, p, len(x))


def fir(x, filt):
    c = np.asarray(filt, dtype=np.float64)
    c = c / abs(np.max(c))
    k = int(round(c.shape[0] / 2))
    y = _shift_left(signal.convolve(x, c, mode="full"), k, len(x))
    ex, ef = float(np.dot(x, x)), float(np.dot(y, y))
    return np.sqrt(ex / ef) * y if ef > 0 else x.copy()


def _segment(wav, beg, n):
    seg = np.zeros(n)
    part = np.asarray(wav, dtype=np.float64)[beg:beg + n]
    seg[:len(part)] = part
    return seg


def _k(x, n, snr):
    ex, en = float(np.dot(x, x)), float(np.dot(n, n))
    return (np.sqrt(ex / ((10 ** (snr / 10.)) * en)) if en > 0 else 1.0), ex, en


def noise(x, wav, beg, snr):
    n = _segment(wav, beg, len(x))
    K, ex, en = _k(x, n, snr)
    if not en > 0:
        return x.copy()
    v = x + K * n
    return np.sqrt(ex / (np.dot(v, v) + 1e-14)) * v


def overlap(x, wav, shift, beg, snr, ir=None):
    T = len(x)
    seg = _segment(wav, beg, T - shift)
    if ir is not None:
        seg = reverb(seg, ir)
    n = np.concatenate([np.zeros(shift), seg])
    K, ex, _ = _k(x, n, snr)
    v = x + K * n
    return np.sqrt(ex / (np.dot(v, v) + 1e-14)) * v


def overlap_label(T, shift, d):
    m = np.concatenate([np.zeros(shift), np.ones(T - shift)])
    return m.reshape(-1, d).mean(1)


def clip(x, cf):
    return np.minimum(np.maximum(x, cf * np.min(x)), cf * np.max(x))


def distort(x, plan, banks):
    """Every stage of `plan` on x (float64, length T), in the reference's order."""
    y = np.asarray(x, dtype=np.float64).copy()
    if "reverb" in plan:
        y = reverb(y, banks["irs"][plan["reverb"]["ir"]])
    if "overlap" in plan:
        d = plan["overlap"]
        ir = banks["irs"][d["ir"]] if "ir" in d else None
        y = overlap(y, banks["overlap"][d["file"]], d["shift"], d["beg"], d["snr"], ir)
    if "noise" in plan:
        d = plan["noise"]
        y = noise(y, banks["noise"][d["file"]], d["beg"], d["snr"])
    if "clip" in plan:
        y = clip(y, plan["clip"]["cf"])
    if "bandrop" in plan:
        y = fir(y, banks["bandrop"][plan["bandrop"]["filt"]])
    if "downsample" in plan:
        y = fir(y, banks["downsample"][plan["downsample"]["filt"]])
    return y
