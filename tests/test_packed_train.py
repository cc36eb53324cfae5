"""WaveFe.encode_packed_train (DESIGN.md section 19) on the CPU with emulated kernels
(tests/emul/): features, per-utterance waveform gradients, parameter gradients,
running statistics and counters against a float64 oracle whose BatchNorms see the
time-concatenation of the utterances; equality with the uniform train forward at equal lengths;
the coupling through the batch statistics; the refusals; the shared plan's generation guard;
no_grad; launches independent of the number of utterances and the zero-row rule."""
import pytest
import torch
import torch.nn.functional as F

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
    cfg = load_golden(MINI[cfg_name])[1]["cfg"] if cfg_name in MINI else cfg_name
    model = WaveFe(**resolve_cfg(cfg))
    model.precision = precision
    sd = fill_state_dict(model.state_dict(), seed)
    for k, v in sd.items():                     # running statistics away from their defaults
        if k.endswith("running_var"):
            sd[k] = v.abs() + 0.5
    model.load_state_dict(sd)
    return model.train()


def buffers(model):
    return {k: v.clone() for k, v in model.named_buffers()}


def run_train(model, wavs, cots, cap=None):
    """encode_packed_train + backward of sum_i <y_i, cot_i> (cot None: no gradient for y_i)."""
    xs = [w.clone().requires_grad_(True) for w in wavs]
    model.zero_grad(set_to_none=True)
    cap = cap or sum(w.numel() for w in wavs) + 4096
    ys = model._encode_packed(xs, cap, CPU, True)
    loss = sum((y * c).sum() for y, c in zip(ys, cots) if c is not None)
    loss.backward()
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    return [y.detach() for y in ys], [x.grad for x in xs], grads


def packed_oracle(xs, sd, cfg, new_stats):
    """float64 train forward of the utterances xs ((1,1,T_i) each): per utterance reflect pad +
    conv, BatchNorm over the time-concatenation of the utterances, PReLU, pooled skips, QRNN and
    the output projection per utterance, norm_out over the concatenation."""
    cfg = O.normalize_fe_cfg(cfg)
    nblk = len(cfg["kwidths"])
    hs, skips = list(xs), [[] for _ in xs]
    for i, (k, s) in enumerate(zip(cfg["kwidths"], cfg["strides"])):
        p = "blocks.%d." % i
        sinc = cfg["sincnet"] and i == 0
        if sinc:
            k += 1 - k % 2
            w, b = O.sinc_filters(sd[p + "conv.low_hz_"], sd[p + "conv.band_hz_"], k, cfg["sr"]), None
        else:
            w, b = sd[p + "conv.weight"], sd[p + "conv.bias"]
        pl, pr = O._pads(k, s, sinc)
        hs = [F.conv1d(F.pad(h, (pl, pr), mode="reflect") if pl + pr else h, w, b, stride=s)
              for h in hs]
        lens = [h.shape[2] for h in hs]
        h = O._bn(torch.cat(hs, 2), sd, p + "norm.", True, new_stats=new_stats)
        hs = list(torch.split(O._prelu(h, sd[p + "act.weight"]), lens, 2))
        if cfg["denseskips"] and i + 1 < nblk:
            for j, h in enumerate(hs):
                skips[j].append(F.conv1d(h, sd["denseskips.%d.weight" % i]))
    if cfg["rnn_pool"]:
        hs = [O._qrnn(h, sd, "rnn.layers.0.") for h in hs]
    ys = []
    for j, h in enumerate(hs):
        y = F.conv1d(h, sd["W.weight"], sd["W.bias"])
        for sk in skips[j]:
            y = y + O._pool_skip(sk, y.shape[2])
        ys.append(y)
    if cfg["norm_out"]:
        lens = [y.shape[2] for y in ys]
        y = O._bn(torch.cat(ys, 2), sd, "norm_out.", True, affine=False, new_stats=new_stats)
        ys = list(torch.split(y, lens, 2))
    return ys


def oracle(model, wavs, cots, before):
    """-> features, dx_i, parameter gradients, new running statistics (float64), from the
    module's parameters and the running statistics `before`."""
    s = {k: (v.double() if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    s.update({k: (v.double() if v.is_floating_point() else v) for k, v in before.items()})
    leaves = {k: s[k].clone().requires_grad_(True) for k, _ in model.named_parameters()}
    s.update(leaves)
    xs = [w.double().view(1, 1, -1).requires_grad_(True) for w in wavs]
    stats = {}
    ys = packed_oracle(xs, s, model.cfg, stats)
    sum((y * c.double()).sum() for y, c in zip(ys, cots) if c is not None).backward()
    return ([y.detach() for y in ys], [x.grad.view(-1) for x in xs],
            {k: v.grad for k, v in leaves.items()}, stats)


def lengths_for(model):
    return [enc.min_length(model.cfg), 1763, 2348]


def check_against_oracle(model, wavs, cots, before, ys, dxs, grads, dx_tol=1e-4):
    rys, rdx, rp, rstats = oracle(model, wavs, cots, before)
    for y, r in zip(ys, rys):
        assert y.shape == r.shape[:1] + r.shape[1:]
        assert rel_l2(y, r) < 1e-4, rel_l2(y, r)
    for dx, r in zip(dxs, rdx):
        assert rel_l2(dx, r) < dx_tol, rel_l2(dx, r)
    gmax = max(float(v.norm()) for v in rp.values())
    for k, v in rp.items():
        if float(v.norm()) < 1e-9 * gmax:   # a bias in front of a train-mode BatchNorm: zero
            assert float(grads[k].norm()) < 1e-5 * gmax, k
            continue
        assert rel_l2(grads[k], v) < 2e-3, (k, rel_l2(grads[k], v))
    now = dict(model.named_buffers())
    for k, v in rstats.items():
        if k.endswith("num_batches_tracked"):
            assert int(now[k]) == int(before[k]) + 1 == int(v), k
        else:
            assert rel_l2(now[k], v) < 1e-5, (k, rel_l2(now[k], v))
    assert set(rstats) == {k for k in now if "running" in k or "num_batches" in k}


@pytest.mark.parametrize("precision", ["fp32", "3xtf32"])
@pytest.mark.parametrize("name,long", [(c, False) for c in CONFIGS] + [("mini", True)])
def test_matches_float64_oracle(name, long, precision, emulated):
    """fold 4 (fp32) and fold 32 (3xtf32) plans; `long` adds an utterance above 512 frames
    (83000 samples: the sequential QRNN scan)."""
    model = make_model(name, precision)
    lens = lengths_for(model) + ([83000] if long else [])
    wavs = [seeded_randn((T,), 100 + T, 0.5) for T in lens]
    shapes = [(1, model.emb_dim, model.frame_counts(T)[-1]) for T in lens]
    cots = [seeded_randn(s, 7 + i) for i, s in enumerate(shapes)]
    before = buffers(model)
    ys, dxs, grads = run_train(model, wavs, cots)
    check_against_oracle(model, wavs, cots, before, ys, dxs, grads)


@pytest.mark.parametrize("n", [1, 3])
def test_equal_lengths_match_uniform_train(n, emulated):
    """n equal lengths: the packed train forward and backward are the uniform train encode of
    the stacked (n, 1, T) batch (features, running statistics, dx, parameter gradients)."""
    T = 2000
    wavs = [seeded_randn((T,), 300 + i, 0.5) for i in range(n)]
    a, b = make_model(CONFIGS[0], "3xtf32"), make_model(CONFIGS[0], "3xtf32")
    shape = (1, a.emb_dim, a.frame_counts(T)[-1])
    cots = [seeded_randn(shape, 40 + i) for i in range(n)]
    ys, dxs, grads = run_train(a, wavs, cots)
    x = torch.stack(wavs).view(n, 1, T).requires_grad_(True)
    out, _ = b._encode(x)
    (out * torch.cat(cots)).sum().backward()
    assert rel_l2(torch.cat(ys), out.detach()) < 1e-6
    assert rel_l2(torch.stack(dxs), x.grad.view(n, T)) < 1e-5
    for k, p in b.named_parameters():
        assert rel_l2(grads[k], p.grad) < 1e-5, k
    bb = dict(b.named_buffers())
    for k, v in a.named_buffers():
        assert rel_l2(v.double(), bb[k].double()) < 1e-6, k


def test_coupling_and_permutation(emulated):
    """A cotangent on one utterance reaches every utterance's dx through the batch statistics
    (as the oracle's); permuting the utterances only reorders the statistics' sums."""
    model = make_model(CONFIGS[0], "3xtf32")
    freeze(model)
    lens = lengths_for(model)
    wavs = [seeded_randn((T,), 200 + T, 0.5) for T in lens]
    shapes = [(1, model.emb_dim, model.frame_counts(T)[-1]) for T in lens]
    cots = [seeded_randn(s, 30 + i) for i, s in enumerate(shapes)]
    before = buffers(model)
    only = [cots[0], None, None]
    _, odx, _ = run_train(model, wavs, only)
    _, rdx, _, _ = oracle(model, wavs, only, before)
    for k in (1, 2):
        assert float(odx[k].abs().max()) > 0.0
        # only the statistics terms reach them, differences of larger fp32 terms: the uniform
        # train backward of a B=3 batch with one cotangent is 4e-4 .. 6e-3 from the oracle there
        assert rel_l2(odx[k], rdx[k]) < 1e-2, rel_l2(odx[k], rdx[k])
    model.load_state_dict({**model.state_dict(), **before})
    ys, dxs, _ = run_train(model, wavs, cots)
    perm = [2, 0, 1]
    model.load_state_dict({**model.state_dict(), **before})
    pys, pdx, _ = run_train(model, [wavs[i] for i in perm], [cots[i] for i in perm])
    for j, i in enumerate(perm):
        assert rel_l2(pys[j], ys[i]) < 1e-6
        assert rel_l2(pdx[j], dxs[i]) < 1e-5


def test_refusals(emulated):
    """Eval mode, a CPU module, a total above max_samples and a short utterance raise before
    any launch and leave the running statistics alone."""
    model = make_model(CONFIGS[0], "fp32")
    m = enc.min_length(model.cfg)
    before = buffers(model)
    n0 = ops.launch_count
    with pytest.raises(RuntimeError, match="CUDA"):
        model.encode_packed_train([torch.zeros(3000)])
    with pytest.raises(ValueError, match="max_samples"):
        model._encode_packed([torch.zeros(3000), torch.zeros(3000)], 5000, CPU, True)
    with pytest.raises(ValueError, match="utterance 1"):
        model._encode_packed([torch.zeros(3000), torch.zeros(m - 1)], 1 << 16, CPU, True)
    model.eval()
    with pytest.raises(RuntimeError, match="encode_packed"):
        model.encode_packed_train([torch.zeros(3000)])
    assert ops.launch_count == n0
    for k, v in model.named_buffers():
        assert torch.equal(v, before[k]), k


def test_generation_guard_shared_plan(emulated):
    """encode_packed and encode_packed_train share the packed plan of a capacity: a forward of
    either between a differentiated forward and its backward makes the backward raise."""
    model = make_model(CONFIGS[0], "fp32")
    xs = [seeded_randn((2000,), 5, 0.5).requires_grad_(True)]
    ys = model._encode_packed(xs, 1 << 15, CPU, True)
    model.eval()
    with torch.no_grad():
        model._encode_packed([seeded_randn((1800,), 6, 0.5)], 1 << 15, CPU)
    with pytest.raises(RuntimeError, match="overwritten"):
        ys[0].sum().backward()
    zs = model._encode_packed(xs, 1 << 15, CPU)
    model.train()
    model._encode_packed([seeded_randn((1800,), 6, 0.5).requires_grad_(True)], 1 << 15, CPU, True)
    with pytest.raises(RuntimeError, match="overwritten"):
        zs[0].sum().backward()


def test_no_grad_updates_statistics(emulated):
    model = make_model("mini", "fp32")
    before = buffers(model)
    wavs = [seeded_randn((T,), T, 0.5) for T in (1500, 2100)]
    with torch.no_grad():
        ys = model._encode_packed([w.requires_grad_(True) for w in wavs], 1 << 14, CPU, True)
    assert all(y.grad_fn is None for y in ys)
    for k, v in model.named_buffers():
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(before[k]) + 1
        else:
            assert not torch.equal(v, before[k]), k


def test_launches_independent_of_count(monkeypatch):
    launches = []

    def counting(name, *args):
        launches.append(name)
        return emul.call(name, *args)

    monkeypatch.setattr(ops, "call", counting)
    model = make_model("mini", "3xtf32")
    counts = []
    for n in (1, 4):
        wavs = [seeded_randn((1200 + 50 * i if i % 2 == 0 else 83000 + 7 * i,), i, 0.5)
                for i in range(n)]
        for frozen in (False, True):
            freeze(model, frozen)
            xs = [w.clone().requires_grad_(True) for w in wavs]
            n0 = ops.launch_count
            ys = model._encode_packed(xs, 1 << 19, CPU, True)
            sum(y.sum() for y in ys).backward()
            counts.append(ops.launch_count - n0)
    assert counts[0] == counts[2] and counts[1] == counts[3], counts


def test_zero_rows_rewritten(emulated):
    """Rows of the backward layout outside the valid frames are zero after a call with other
    offsets, even after a call that left NaN there."""
    model = make_model(CONFIGS[0], "fp32")
    freeze(model)
    wavs = [seeded_randn((T,), T, 0.5) for T in (1500, 2100, 900)]
    before = buffers(model)
    _, dx_ref, _ = run_train(model, wavs, [torch.ones(1) for _ in wavs], 1 << 14)
    plan = model._grad_plan(1 << 14, CPU)
    for t in plan.dyz + [plan.dYg]:
        t.fill_(float("nan"))
    run_train(model, wavs[::-1], [torch.ones(1) for _ in wavs], 1 << 14)
    model.load_state_dict({**model.state_dict(), **before})
    _, dx, _ = run_train(model, wavs, [torch.ones(1) for _ in wavs], 1 << 14)
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
