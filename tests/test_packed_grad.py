"""WaveFe.encode_packed (DESIGN.md section 18) on the CPU with emulated kernels
(tests/emul/): per-utterance waveform gradients and summed parameter gradients
against float64 autograd through the oracle, independence from the neighbours in the pack, the
refusals, the generation guard, launches independent of the number of utterances and the
zero-row rule of the backward layout."""
import pytest
import torch

import emul
import pase_oracle as O
from helpers import load_golden, resolve_cfg, fill_state_dict, seeded_randn, rel_l2
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import WaveFe

CPU = torch.device("cpu")
CONFIGS = ["cfg/frontend/PASE+.cfg", "cfg/frontend/PASE.cfg", "mini", "mininornn"]
MINI = {"mini": "enc_mini_train_1763", "mininornn": "enc_mininornn_train_1600"}


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "call", emul.call)
    yield


def freeze(model, frozen=True):
    for _, p in model.named_parameters():
        p.requires_grad_(not frozen)


def make_model(cfg_name, precision, seed=11):
    """A config file, or one of the two mini configs of the goldens (MINI)."""
    cfg = load_golden(MINI[cfg_name])[1]["cfg"] if cfg_name in MINI else cfg_name
    model = WaveFe(**resolve_cfg(cfg))
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    return model.eval()


def run_packed(model, wavs, cots, cap=None):
    """encode_packed + backward of sum_i <y_i, cot_i> (cot None: no gradient for y_i)."""
    xs = [w.clone().requires_grad_(True) for w in wavs]
    model.zero_grad(set_to_none=True)
    cap = cap or sum(w.numel() for w in wavs) + 4096
    ys = model._encode_packed(xs, cap, CPU)
    loss = sum((y * c).sum() for y, c in zip(ys, cots) if c is not None)
    loss.backward()
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    return ys, [x.grad for x in xs], grads


def oracle(model, w, cot):
    """float64 dx and parameter gradients of <y, cot> for one utterance alone."""
    sd = model.state_dict()
    s = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    leaves = {k: s[k].clone().requires_grad_(True) for k, _ in model.named_parameters()}
    s.update(leaves)
    x = w.double().view(1, 1, -1).requires_grad_(True)
    y = O.encoder_forward(x, s, model.cfg, training=False)
    (y * cot.double()).sum().backward()
    return x.grad.view(-1), {k: v.grad for k, v in leaves.items()}


def lengths_for(model):
    m = enc.min_length(model.cfg)
    return [m, 1763, 2345 + 3]            # the shortest, a length that is no multiple of 32


@pytest.mark.parametrize("precision", ["fp32", "3xtf32"])
@pytest.mark.parametrize("name,long", [(c, False) for c in CONFIGS] + [("mini", True)])
def test_matches_float64_oracle(name, long, precision, emulated):
    """fold 4 (fp32) and fold 32 (3xtf32) plans; `long` adds an utterance above 512 frames
    (83000 samples: the sequential QRNN scan) to one below."""
    model = make_model(name, precision)
    lens = lengths_for(model) + ([83000] if long else [])
    if long:
        assert model.frame_counts(83000)[-1] > 512 >= model.frame_counts(lens[-2])[-1]
    wavs = [seeded_randn((T,), 100 + T, 0.5) for T in lens]
    with torch.no_grad():
        shapes = [y.shape for y in model._encode_packed(wavs, sum(lens) + 4096, CPU)]
    cots = [seeded_randn(tuple(s), 7 + i) for i, s in enumerate(shapes)]
    ys, dxs, grads = run_packed(model, wavs, cots)
    ref_p = {}
    for w, c, dx in zip(wavs, cots, dxs):
        rdx, rp = oracle(model, w, c)
        assert rel_l2(dx, rdx) < 1e-4, rel_l2(dx, rdx)
        for k, v in rp.items():
            ref_p[k] = v if k not in ref_p else ref_p[k] + v
    for k, v in ref_p.items():
        if float(v.norm()) == 0.0:
            continue
        assert rel_l2(grads[k], v) < 2e-3, (k, rel_l2(grads[k], v))


def test_independent_of_neighbours(emulated):
    model = make_model(CONFIGS[0], "3xtf32")
    freeze(model)
    lens = lengths_for(model)
    wavs = [seeded_randn((T,), 200 + T, 0.5) for T in lens]
    with torch.no_grad():
        shapes = [y.shape for y in model._encode_packed(wavs, 1 << 16, CPU)]
    cots = [seeded_randn(tuple(s), 30 + i) for i, s in enumerate(shapes)]
    _, dxs, _ = run_packed(model, wavs, cots)
    perm = [2, 0, 1]
    _, pdx, _ = run_packed(model, [wavs[i] for i in perm], [cots[i] for i in perm])
    for j, i in enumerate(perm):
        assert rel_l2(pdx[j], dxs[i]) < 1e-6
    for i in range(3):
        only = [c if k == i else None for k, c in enumerate(cots)]
        _, odx, _ = run_packed(model, wavs, only)
        assert rel_l2(odx[i], dxs[i]) < 1e-6
        for k in range(3):
            if k != i:
                assert float(odx[k].abs().max()) == 0.0


def test_refusals(emulated):
    model = make_model(CONFIGS[0], "fp32")
    m = enc.min_length(model.cfg)
    with pytest.raises(ValueError, match="split"):
        model._encode_packed([torch.zeros(3000), torch.zeros(3000)], 5000, CPU)
    with pytest.raises(ValueError, match="utterance 1"):
        model._encode_packed([torch.zeros(3000), torch.zeros(m - 1)], 1 << 16, CPU)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.encode_packed([torch.zeros(3000)])
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        model.encode_packed([torch.zeros(3000)])


@pytest.mark.parametrize("second", ["differentiated", "no_grad", "frozen"])
def test_generation_guard(second, emulated):
    """Any later forward on the same plan before the backward makes the backward raise: a
    differentiated one, one under no_grad, and one of a frozen model whose waveforms need no
    gradient (the clean targets of a feature loss)."""
    model = make_model(CONFIGS[0], "fp32")
    freeze(model, second == "frozen")
    xs = [seeded_randn((2000,), 5, 0.5).requires_grad_(True)]
    ys = model._encode_packed(xs, 1 << 15, CPU)
    other = [seeded_randn((1800,), 6, 0.5)]
    if second == "differentiated":
        model._encode_packed([other[0].requires_grad_(True)], 1 << 15, CPU)
    elif second == "no_grad":
        with torch.no_grad():
            model._encode_packed(other, 1 << 15, CPU)
    else:
        model._encode_packed(other, 1 << 15, CPU)
    with pytest.raises(RuntimeError, match="overwritten"):
        ys[0].sum().backward()


def test_launches_independent_of_count(monkeypatch):
    launches = []

    def counting(name, *args):
        launches.append(name)
        return emul.call(name, *args)

    monkeypatch.setattr(ops, "call", counting)
    model = make_model("mini", "3xtf32")
    counts = []
    for n in (1, 4):
        # lengths on both sides of 512 frames: each scan kernel sees utterances of its own
        wavs = [seeded_randn((1200 + 50 * i if i % 2 == 0 else 83000 + 7 * i,), i, 0.5)
                for i in range(n)]
        for frozen in (False, True):
            freeze(model, frozen)
            xs = [w.clone().requires_grad_(True) for w in wavs]
            n0 = ops.launch_count
            ys = model._encode_packed(xs, 1 << 19, CPU)
            sum(y.sum() for y in ys).backward()
            counts.append(ops.launch_count - n0)
    assert counts[0] == counts[2] and counts[1] == counts[3], counts


def test_zero_rows_rewritten(emulated):
    """Rows of the backward layout outside the valid frames read by a GEMM are zero after a call
    with other offsets, even after a call that left garbage there."""
    model = make_model(CONFIGS[0], "fp32")
    freeze(model)
    wavs = [seeded_randn((T,), T, 0.5) for T in (1500, 2100, 900)]
    _, dx_ref, _ = run_packed(model, wavs, [torch.ones(1) for _ in wavs], 1 << 14)
    plan = model._grad_plan(1 << 14, CPU)
    for t in plan.dyz + [plan.dYg]:
        t.fill_(float("nan"))
    _, dx, _ = run_packed(model, wavs[::-1], [torch.ones(1) for _ in wavs], 1 << 14)
    _, dx, _ = run_packed(model, wavs, [torch.ones(1) for _ in wavs], 1 << 14)
    for a, b in zip(dx, dx_ref):
        assert torch.equal(a, b)
    sec, sz = plan.layout
    for l, g in enumerate(plan.geoms):
        C = g.Cout
        rows = plan.table[sec[("bwd", l)]:sec[("bwd", l)] + 9 * 3].view(3, 9).tolist()
        d = plan.dyz[l]
        lead = sz["lead"][l]
        valid = torch.zeros(d.numel(), dtype=torch.bool)
        for T, _, _, _, _, _, _, d_off, span in rows:
            valid[d_off:d_off + T * C] = True
        end = rows[-1][7] + rows[-1][8] * C
        inside = d[rows[0][7] - lead * C:end]
        assert not torch.isnan(inside).any()
        assert float(inside[~valid[rows[0][7] - lead * C:end]].abs().max()) == 0.0
