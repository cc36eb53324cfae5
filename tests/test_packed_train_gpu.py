"""WaveFe.encode_packed_train on one H100 (DESIGN.md section 19): equal lengths against the
uniform train encode, benchmark scale against the float64 oracle of the concatenated-batch
BatchNorms, the frozen sweep and grad_sink, a three-step fine-tuning loop with FlatAdam against
the same steps through the oracle, and allocations after warm-up."""
import pytest
import torch

from helpers import resolve_cfg, fill_state_dict, seeded_randn, rel_l2
from pase_b200.frontend import WaveFe
from pase_b200.optim import FlatAdam
from test_packed_train import packed_oracle

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "3xtf32", "3xf16", "bf16"]
CONFIGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
# equal lengths, packed against uniform: the fp64 statistics are summed by atomics in another
# order, so S1 / S2 / mean can differ in their last fp32 bit; the tf32 and bf16 GEMM operands
# round dy to 10 and 7 mantissa bits, where such a bit flips the rounding of whole channels
# (measured on an H100: <= 2e-6 in fp32, 3xtf32, 3xf16; 4.7e-4 tf32; 6.7e-3 bf16)
GRAD_TOL = {"fp32": 1e-5, "3xtf32": 1e-5, "3xf16": 1e-5, "tf32": 2e-3, "bf16": 2e-2}


def _model(cfg_name, precision):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.precision = precision
    m.load_state_dict(fill_state_dict(m.state_dict(), 11))
    return m.cuda().train()


def _corpus(lengths, seed=5):
    return [seeded_randn((T,), seed + i, 0.5).cuda() for i, T in enumerate(lengths)]


def _packed(m, wavs, cots):
    xs = [w.clone().requires_grad_(True) for w in wavs]
    m.zero_grad(set_to_none=True)
    ys = m.encode_packed_train(xs)
    sum((y * c).sum() for y, c in zip(ys, cots)).backward()
    return ys, [x.grad for x in xs], {k: p.grad.clone() for k, p in m.named_parameters()
                                      if p.grad is not None}


def freeze(m, frozen=True):
    for _, p in m.named_parameters():       # Model.parameters() yields trainable ones only
        p.requires_grad_(not frozen)


def _shapes(m, lengths):
    return [(1, m.emb_dim, m.frame_counts(T)[-1]) for T in lengths]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", CONFIGS)
def test_equal_lengths_match_uniform_train(name, precision):
    """B=8 utterances of 32000 samples: the packed train forward and backward against the
    uniform train encode of the (8, 1, 32000) batch.  Only the order of the fp64 atomic sums of
    the statistics differs."""
    N, T = 8, 32000
    a, b = _model(name, precision), _model(name, precision)
    wavs = _corpus([T] * N, seed=20)
    cots = [seeded_randn(s, 50 + i).cuda() for i, s in enumerate(_shapes(a, [T] * N))]
    ys, dxs, grads = _packed(a, wavs, cots)
    x = torch.stack(wavs).view(N, 1, T).requires_grad_(True)
    b.zero_grad(set_to_none=True)
    out, _ = b.encode(x)
    (out * torch.cat(cots)).sum().backward()
    e_y = rel_l2(torch.cat([y.detach() for y in ys]), out.detach())
    e_dx = rel_l2(torch.stack(dxs), x.grad.view(N, T))
    gmax = max(float(p.grad.norm()) for _, p in b.named_parameters())
    # biases in front of a train-mode BatchNorm have zero gradient up to rounding: skipped
    e_p = max(rel_l2(grads[k], p.grad) for k, p in b.named_parameters()
              if float(p.grad.norm()) > 1e-6 * gmax)
    bb = dict(b.named_buffers())
    e_s = max(rel_l2(v.double(), bb[k].double()) for k, v in a.named_buffers())
    print("%s %s equal lengths: features %.2e, dx %.2e, parameter gradients %.2e, running "
          "statistics %.2e" % (name, precision, e_y, e_dx, e_p, e_s))
    assert e_y <= 1e-6 and e_s <= 1e-6
    assert e_dx <= GRAD_TOL[precision] and e_p <= GRAD_TOL[precision]


def _oracle_steps(m, wavs, cots, dtype):
    """dx (concatenated), parameter gradients and new running statistics of sum_i <y_i, cot_i>
    through the concatenated-batch oracle in `dtype` (plain torch on the device, TF32 off)."""
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    leaves = {k: sd[k].clone().requires_grad_(True) for k, _ in m.named_parameters()}
    sd.update(leaves)
    allow = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        xs = [w.to(dtype).view(1, 1, -1).requires_grad_(True) for w in wavs]
        ys = packed_oracle(xs, sd, m.cfg, {})
        sum((y * c.to(dtype)).sum() for y, c in zip(ys, cots)).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = allow
    return torch.cat([x.grad.view(-1) for x in xs]), {k: v.grad for k, v in leaves.items()}


def _worst(grads, ref):
    gmax = max(float(v.norm()) for v in ref.values())       # biases before a BatchNorm: zero
    return max((rel_l2(grads[k], v), k) for k, v in ref.items() if float(v.norm()) > 1e-9 * gmax)


@pytest.mark.parametrize("precision,floor", [("3xf16", 2e-3), ("3xtf32", 2e-3), ("tf32", 1e-1),
                                             ("bf16", 3e-1)])
def test_benchmark_scale_against_float64_oracle(precision, floor):
    """32 utterances of 24000-40000 samples in one pack against the float64 oracle: dx and each
    parameter gradient within max(2 x the float32 oracle's own error, floor) relative L2.  The
    train-mode BatchNorm backward subtracts the statistics terms, so the float32 oracle's own
    error is larger than in eval mode (section 18's fixed 2e-3 for parameter gradients becomes
    this rule).  tf32 and bf16 round the operands to 10 and 7 mantissa bits: floors 1e-1 and 3e-1
    (measured on an H100: 4.1e-2 / 4.9e-2 and 1.2e-1 / 1.5e-1 for dx / parameters)."""
    g = torch.Generator().manual_seed(9)
    d = (torch.randint(-8000, 8001, (16,), generator=g)).tolist()
    lens = [32000 + x for x in d] + [32000 - x for x in d]
    m = _model(CONFIGS[1], precision)
    wavs = _corpus(lens, seed=70)
    cots = [seeded_randn(s, 90 + i).cuda() for i, s in enumerate(_shapes(m, lens))]
    state = {k: v.clone() for k, v in m.state_dict().items()}
    _, dxs, grads = _packed(m, wavs, cots)
    m.load_state_dict(state)                   # the oracle starts from the same statistics
    d64, p64 = _oracle_steps(m, wavs, cots, torch.float64)
    d32, p32 = _oracle_steps(m, wavs, cots, torch.float32)
    e_dx, e_ref = rel_l2(torch.cat(dxs), d64), rel_l2(d32, d64)
    (e_p, k), (e_pref, kref) = _worst(grads, p64), _worst(p32, p64)
    print("%s B=32 train scale: dx rel-L2 %.2e (float32 oracle %.2e), parameter gradients %.2e "
          "(%s; float32 oracle %.2e, %s)" % (precision, e_dx, e_ref, e_p, k, e_pref, kref))
    assert e_dx <= max(2 * e_ref, floor)
    assert e_p <= max(2 * e_pref, floor)


@pytest.mark.parametrize("precision", ["3xf16", "bf16"])
def test_frozen_sweep_and_sink(precision):
    m = _model(CONFIGS[1], precision)
    lens = [16001, 82081, 3200, 40000]
    wavs = _corpus(lens)
    cots = [seeded_randn(s, 60 + i).cuda() for i, s in enumerate(_shapes(m, lens))]
    _, dx_full, grads = _packed(m, wavs, cots)
    freeze(m)
    runs = [_packed(m, wavs, cots)[1] for _ in range(2)]
    for a, b, c in zip(dx_full, *runs):
        assert torch.equal(a, b) and torch.equal(b, c)
    freeze(m, False)
    opt = FlatAdam([p for _, p in m.named_parameters()], lr=1e-3).bind_encoder(m)
    opt.zero_grad(set_to_none=True)
    xs = [w.clone().requires_grad_(True) for w in wavs]
    sum((y * c).sum() for y, c in zip(m.encode_packed_train(xs), cots)).backward()
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, grads[k]), k
    m.grad_sink = None




def test_fine_tuning_loop_against_float64_oracle():
    """Three FlatAdam steps of PASE+ (3xtf32) and a linear head on mean-pooled features over
    variable-length utterances, against the same steps through the float64 oracle with
    torch.optim.Adam: losses and encoder parameters within 1e-4 relative.  Fine-tuning learning
    rates (1e-5 encoder, 1e-4 head): Adam's first steps are lr * sign(g), so an element whose
    gradient is within rounding of zero moves by +-lr on either side."""
    m = _model(CONFIGS[1], "3xtf32")
    lens = [8000, 23456, 16001, 12000, 31999, 9001]
    wavs = _corpus(lens, seed=33)
    labels = torch.tensor([0, 1, 2, 3, 1, 0], device="cuda")
    head = torch.nn.Linear(m.emb_dim, 4).cuda()
    torch.nn.init.normal_(head.weight, std=0.1, generator=torch.Generator("cuda").manual_seed(3))
    ref_state = {k: v.double().clone() for k, v in m.state_dict().items()}
    ref_head = [p.detach().double().clone().requires_grad_(True) for p in head.parameters()]
    ref_leaves = {k: ref_state[k].clone().requires_grad_(True) for k, _ in m.named_parameters()}
    # a bias in front of a train-mode BatchNorm does not reach the loss: its gradient is rounding
    # noise, which Adam would turn into full-size steps, so it gets learning rate 0 on both sides
    idle = {k for k in ref_leaves if k.endswith("conv.bias") or k == "W.bias"}
    groups = lambda named: [{"params": [p for k, p in named if k not in idle]},
                            {"params": [p for k, p in named if k in idle], "lr": 0.0}]
    ref_opt = torch.optim.Adam(groups(list(ref_leaves.items()))
                               + [{"params": ref_head, "lr": 1e-4}], lr=1e-5)

    opt = FlatAdam(groups(list(m.named_parameters())), lr=1e-5).bind_encoder(m)
    hopt = torch.optim.Adam(head.parameters(), lr=1e-4)
    allow = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for step in range(3):
            opt.zero_grad(set_to_none=True)
            hopt.zero_grad(set_to_none=True)
            feats = m.encode_packed_train(wavs)
            pooled = torch.cat([f.mean(2) for f in feats])
            loss = torch.nn.functional.cross_entropy(head(pooled), labels)
            loss.backward()
            opt.step()
            hopt.step()

            ref_opt.zero_grad(set_to_none=True)
            sd = dict(ref_state)
            sd.update(ref_leaves)
            stats = {}
            ys = packed_oracle([w.double().view(1, 1, -1) for w in wavs], sd, m.cfg, stats)
            rp = torch.cat([y.mean(2) for y in ys])
            rloss = torch.nn.functional.cross_entropy(rp @ ref_head[0].t() + ref_head[1], labels)
            rloss.backward()
            ref_opt.step()
            ref_state.update({k: v.detach() for k, v in stats.items()})
            e_loss = abs(float(loss) - float(rloss)) / abs(float(rloss))
            e_par, k = max((rel_l2(p.detach(), ref_leaves[k].detach()), k)
                           for k, p in m.named_parameters())
            print("step %d: loss %.6f (oracle %.6f, rel %.1e), parameters rel-L2 %.1e (%s)"
                  % (step, float(loss.detach()), float(rloss.detach()), e_loss, e_par, k))
            assert e_loss < 1e-4 and e_par < 1e-4
    finally:
        torch.backends.cudnn.allow_tf32 = allow
        m.grad_sink = None
    for k, v in m.named_buffers():
        if "running" in k:
            assert rel_l2(v.double(), ref_state[k]) < 1e-4, k


def _r512(nbytes):
    return -(-nbytes // 512) * 512          # the caching allocator's block granularity


@pytest.mark.parametrize("frozen", [False, True])
def test_allocations_after_warmup(frozen):
    """After warm-up a call keeps nothing allocated but its outputs (one buffer), the packed dx
    and, in the full sweep, the parameter gradients (as section 18's bound)."""
    m = _model(CONFIGS[1], "3xf16")
    freeze(m, frozen)
    lens = [471, 16001, 82081, 3200]
    wavs = _corpus(lens)
    cots = [torch.randn(s, device="cuda") for s in _shapes(m, lens)]
    for _ in range(2):
        _packed(m, wavs, cots)
    m.zero_grad(set_to_none=True)
    xs = [w.clone().requires_grad_(True) for w in wavs]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    ys = m.encode_packed_train(xs)
    sum((y * c).sum() for y, c in zip(ys, cots)).backward()
    torch.cuda.synchronize()
    bound = _r512(sum(y.numel() for y in ys) * 4) + _r512(sum(w.numel() for w in wavs) * 4)
    if not frozen:
        plan = next(iter(m._grad_plans.values()))
        params = [p for _, p in m.named_parameters()]
        bound += sum(_r512(p.numel() * 4) for p in params) + _r512(plan.grad_vec.numel() * 4)
        bound += _r512(sum(p.numel() * 4 for n, p in m.named_parameters()
                           if n.endswith("conv.weight") and p.dim() == 3))
        assert all(p.grad is not None for p in params)
    grew = torch.cuda.memory_allocated() - base
    print("frozen=%s: %d bytes kept, bound %d" % (frozen, grew, bound))
    assert grew <= bound
