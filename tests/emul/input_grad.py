"""The input-gradient entry points (pase_sinc_dgrad_pack, pase_sinc_dgrad_weight,
pase_reflect_fold_wave) that the encoder's backward launches when the waveform needs a
gradient."""
import torch

from .core import _as, _reflect


def pase_sinc_dgrad_pack(src, src_lo, dst, dst_lo, esz, N, C, T_out, src_frames, halo,
                         dst_frames):
    assert (src_lo is None) == (dst_lo is None) and src.element_size() == esz
    for s, d in ((src, dst), (src_lo, dst_lo)):
        if d is None:
            continue
        out = torch.zeros(N, dst_frames, C, dtype=d.dtype)
        out[:, halo:halo + T_out] = _as(s, (N, T_out, C), (src_frames * C, C, 1))
        d[:N * dst_frames * C] = out.reshape(-1)


def sinc_dgrad_operand(filt, C, k, fold, rows):
    """(fold, rows*fold, C) banded operand: [p, r*fold+q, co] = filt[co][H+p-fold*r-q]."""
    H = (rows - 1) * fold
    f = filt[:C * k].view(C, k)
    j = H + torch.arange(fold)[:, None] - torch.arange(rows * fold)[None, :]
    valid = (j >= 0) & (j < k)
    w = f[:, j.clamp(0, k - 1)].permute(1, 2, 0)
    return torch.where(valid[:, :, None], w, torch.zeros_like(w))


def pase_sinc_dgrad_weight(filt, Wdg, C, k, fold, rows):
    assert (rows - 1) * fold >= k - 1
    Wdg[:fold * rows * fold * C] = sinc_dgrad_operand(filt, C, k, fold, rows).reshape(-1)


def reflect_fold(dpad, N, T, padL, padR):
    """float64 adjoint of the reflect pad: (N, T+padL+padR) -> (N, T)."""
    idx = _reflect(torch.arange(T + padL + padR) - padL, T)
    out = torch.zeros(N, T, dtype=torch.float64)
    out.index_add_(1, idx, dpad.double())
    return out


def pase_reflect_fold_wave(dpad, pitch, dx, N, T, padL, padR):
    d = _as(dpad, (N, T + padL + padR), (pitch, 1))
    dx[:N * T] = reflect_fold(d, N, T, padL, padR).float().reshape(-1)
