"""The references, bounds and table constructions of tests/test_packed_kernels_gpu.py run on the
CPU against the fp32 emulations the CPU suite uses in place of the packed and windowed kernels
(tests/emul/packed.py, tests/emul/windowed.py), and the host-side layout invariants those
kernels rely on: every padded operand starts on a folded-row boundary, every utterance's zero
tail covers the next one's halo, table values stay below INDEX_LIMIT, and no pack holds more
utterances than a launch grid has rows.  Bit equality with the uniform kernels and the tensor-core tail plan depend on
the hardware and stay in the GPU file."""
import numpy as np
import pytest
import torch

import pase_b200.ops as ops
from pase_b200 import encoder as E
import test_packed_kernels_gpu as K
from test_packed_train import CPU, buffers, emulated, make_model  # noqa: F401
from test_qrnn_sinc_out_gpu import _check_all, _report, _within

DEV = "cpu"


# ---- host-level layout invariants ----
@pytest.mark.parametrize("prec", ["fp32", "3xtf32", "bf16", "3xf16"])
@pytest.mark.parametrize("key", ["edges", "seeded48", "single"])
def test_layout_invariants(key, prec):
    lengths = K.length_lists(K.pasep_cfg())[key]
    plan, geoms, host, sec, sz = K.product_layout(lengths, prec)
    n, G = len(lengths), plan.geoms
    assert host.max() < E.INDEX_LIMIT and host.min() >= 0
    assert n <= plan.max_utts <= E.MAX_UTTS
    wave = host[sec["wave"]:sec["wave"] + 3 * n].reshape(n, 3)
    assert (wave[:, 0] == np.concatenate([[0], np.cumsum(lengths)])[:n]).all()
    assert (wave[:, 2] % G[0].lda == 0).all(), "waveform operand off a folded-row boundary"
    for l, g in enumerate(G):
        row0, orow0, tv = K._var_rows(host[sec[("gemm", l)]:], n)
        assert (np.diff(row0) == [gi[l].P for gi in geoms]).all()
        assert (tv == [gi[l].T_out for gi in geoms]).all()
        assert row0[-1] == sz["gemm_rows"][l]
        for gi in geoms:
            if g.sinc:          # P folded rows of fold samples
                assert gi[l].fold * gi[l].P - gi[l].T_out >= g.k - 1, "sinc tail < halo"
            else:
                assert gi[l].P - gi[l].T_out >= gi[l].taps - 1, "zero tail shorter than the halo"
        if l + 1 < plan.nblk:
            bn = host[sec[("bn", l)]:sec[("bn", l)] + 6 * n].reshape(n, 6)
            nx = G[l + 1]
            assert (bn[:, 2] % nx.lda == 0).all(), "block %d operand off a row boundary" % (l + 1)
            next_row0 = K._var_rows(host[sec[("gemm", l + 1)]:], n)[0][:n]
            assert (bn[:, 2] // nx.lda == next_row0).all()
            assert (bn[:, 5] * bn[:, 4] <= bn[:, 0]).all(), "pool_T * pool_d > T"


def test_split_packs_respects_the_grid_row_limit():
    """70 000 clips of 471 samples under max_samples = 33 000 000 (below INDEX_LIMIT): no pack
    above 65 535 utterances; an explicit count splits further; a count past the limit raises."""
    lengths = [471] * 70000
    packs = E.split_packs(lengths, 33_000_000)
    assert max(b - a for a, b in packs) == E.MAX_UTTS == K.MAX_GRID_Y
    assert packs[0] == (0, E.MAX_UTTS) and packs[-1][1] == 70000
    assert E.split_packs([4, 4, 4, 4, 4], 100, 2) == [(0, 2), (2, 4), (4, 5)]
    assert E.split_packs([4, 20, 4], 8, 1) == [(0, 1), (1, 2), (2, 3)]
    for bad in (0, E.MAX_UTTS + 1):
        with pytest.raises(ValueError, match="max_count"):
            E.split_packs(lengths, 1 << 30, bad)


def test_packed_plan_caps_utterances():
    """A capacity that holds more minimum-length utterances than a grid has rows."""
    cfg = make_model("mini", "fp32").cfg
    cap = (E.MAX_UTTS + 1000) * E.min_length(cfg)
    plan = E.PackedPlan(cfg, cap, torch.device("meta"), "fp32")
    assert plan.max_utts == E.MAX_UTTS
    assert E.PackedPlan(cfg, 10 * E.min_length(cfg), torch.device("meta")).max_utts == 10


@pytest.mark.parametrize("train", [False, True])
def test_encode_packed_refuses_more_utterances_than_a_pack(train, emulated):  # noqa: F811
    model = make_model("mini", "fp32")
    if not train:
        model.eval()
    m = E.min_length(model.cfg)
    wavs = list(torch.zeros((E.MAX_UTTS + 1) * m).split(m))
    before = buffers(model)
    n0 = ops.launch_count
    with pytest.raises(ValueError, match="65536 utterances exceed the 65535"):
        model._encode_packed(wavs, len(wavs) * m, CPU, train)
    assert ops.launch_count == n0
    for k, v in model.named_buffers():
        assert torch.equal(v, before[k]), k


# ---- the GPU file's references and bounds against the emulations ----
def _emulated_cases():
    out = []
    for name in ("ffma-conv1-edges", "tf32-conv2-edges", "3xf16-conv2-edges-c16-oddldc"):
        v, C, cs, cq = K.gemm_case(name, DEV, True)
        out += v.checks(C, cs, cq)
    lists = K.length_lists(K.pasep_cfg())
    for key in ("edges", "single"):
        w = K.Wave(lists[key], 125, 125, DEV)
        for fmt in (0, 1, 2):
            out += K.pad_checks(w, fmt)[2]
        out += K.fold_checks(w)[1]
    out += K.fold_acc_checks(DEV)
    Ts = [3, 48, 20, 1]
    for prec in K.BN_PRECS:             # each utterance its own pool_T, frames left unpooled
        b = K.BnVar(Ts, 16, DEV, K.pool_rule(Ts, [1, 5, 6, 1]), prec=prec, seed=1)
        out += K.bn_fwd_checks(b, sep=1, pool=True)[4]
        b3 = K.BnVar(Ts[:3], 16, DEV, K.pool_rule(Ts[:3], [1, 5, 6]), prec=prec, seed=2)
        out += K.bn_fwd_checks(b3, sep=0, pool=False, padL=2, padR=2)[4]
        train, amax, r = K.bn_reduce_checks(b)
        out += r
        dst, lo, db, so = b.apply(amax=amax)
        out += K.bn_apply_checks(b, dst, db, lo=lo, so=so)
        dst, lo, db, so = b.apply(train=train, amax=amax)
        out += K.bn_apply_checks(b, dst, db, train, lo=lo, so=so)
    q = K.QrnnVar((1, 16, 17, 40), 12, DEV, seed=3)
    q.run()
    out += q.checks(True)
    out += K.qrnn_carry_checks(DEV, H=6)[0]
    o = K.OutVar([1, 7, 30, 3], 12, DEV, seed=4)
    for mode in (0, 1, 2, 3):
        out += K.out_affine_var_checks(o, mode)
    for mode in (1, 2, 3):
        out += K.out_place_select_checks(o, mode)
    out += K.out_bwd_checks(o)
    K.stream_gather_checks(DEV)
    return out


def test_bounds_hold_for_emulation():
    checks = _emulated_cases()
    _report("packed emulation", _check_all(checks))
    tested = 0
    for w, got, ref, tol in checks:
        tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(got).reshape(-1)
        if not bool((tol > 0).any()):
            continue
        i = int(torch.argmax(tol))         # the loosest element of the check: moved past it
        bumped = got.double().reshape(-1).clone()
        bumped[i] += 2 * tol[i]
        with pytest.raises(AssertionError, match="out of bound"):
            _within(w, bumped.view(got.shape), ref, tol.view(got.shape))
        tested += 1
    assert tested >= 30, tested
