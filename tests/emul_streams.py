"""TEST-ONLY torch emulation of the StreamPool entry points (include/pase_b200.h:
pase_stream_gather, pase_qrnn_scan_fwd_carry_var, pase_out_place_var); each row of a table runs
the emulation of the one-stream entry point it generalises (tests/emul_long.py), and every other
entry point goes to tests/emul_long.py."""
import torch

import emul_long


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
        emul_long.pase_qrnn_scan_fwd_carry(Y[row0 * 3 * H:], h[row0 * ldh:], ldh, Cst[row0 * H:],
                                           None if first else st, st, T, H)


def pase_out_place_var(y, scale, shift, out, tab, nseg, max_T, C):
    for row0, T, ocol, ldo, col0 in _rows(tab, nseg, 5):
        assert T <= max_T
        emul_long.pase_out_place(y[row0 * C:], scale, shift, out[ocol * C:], ldo, col0, T, C)


def call(name, *args):
    fn = globals().get(name)
    if fn is None:
        return emul_long.call(name, *args)
    with torch.no_grad():
        fn(*args)
    return 0
