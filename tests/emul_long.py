"""TEST-ONLY torch emulation of the windowed long-recording entry points (include/pase_b200.h:
pase_qrnn_scan_fwd_carry, pase_out_place, pase_out_select); every other entry point goes to the
packed / uniform emulations (tests/emul_extract.py, tests/emul_ops.py)."""
import torch

import emul_extract
from pase_b200.modules import select_output

_MODES = {1: "avg_norm", 2: "avg_concat", 3: "avg_norm_concat"}


def pase_qrnn_scan_fwd_carry(Y, h, ldh, Cst, c_in, c_out, T, H):
    y = Y[:T * 3 * H].view(T, 3 * H)
    z, f, o = torch.tanh(y[:, :H]), torch.sigmoid(y[:, H:2 * H]), torch.sigmoid(y[:, 2 * H:])
    c = torch.zeros(H) if c_in is None else c_in[:H].clone()
    for t in range(T):
        c = f[t] * z[t] + (1 - f[t]) * c
        Cst[t * H:(t + 1) * H] = c
        h[t * ldh:t * ldh + H] = o[t] * c
    c_out[:H] = c


def pase_out_place(y, scale, shift, out, ldo, col0, T, C):
    # one rounding of y*scale + shift, as the kernel's fmaf
    v = (y[:T * C].view(T, C).double() * scale[:C].double() + shift[:C].double()).float()
    out.view(-1)[:C * ldo].view(C, ldo)[:, col0:col0 + T] = v.t()


def pase_out_select(out, T, C, mode):
    o = out.view(-1)
    h = o[:C * T].view(1, C, T).clone()
    f = select_output(h.double(), _MODES[mode]).float()
    o[:f.numel()] = f.reshape(-1)


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        return emul_extract.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
