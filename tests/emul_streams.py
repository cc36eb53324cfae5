"""TEST-ONLY torch emulation of the windowed entry points (include/pase_b200.h:
pase_stream_gather, pase_qrnn_scan_fwd_carry_var, pase_out_place_var, pase_out_select) that
StreamPool, and so FeatureStream and WaveFe.extract_long, launch; every other entry point goes to
the packed / uniform emulations (tests/emul_extract.py, tests/emul_ops.py)."""
import torch

import emul_extract
from pase_b200.modules import select_output

_MODES = {1: "avg_norm", 2: "avg_concat", 3: "avg_norm_concat"}


def _rows(tab, n, width):
    return tab[:n * width].view(n, width).tolist()


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


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        return emul_extract.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
