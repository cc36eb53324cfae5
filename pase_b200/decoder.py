"""Transposed-convolution stack of the ``cchunk`` DecoderMinion (GDeconv1DBlock,
modules.py:558-589; workers+.cfg:3-14) as polyphase GEMMs over channel-last rows.

ConvTranspose1d(k, stride s, padding p):  y[s*u+q-p] = sum_v x[u-v] . W[:, :, s*v+q].
Row u of the GEMM reads `taps = ceil(k/s)` consecutive input frames (an overlapping
view of the zero-padded input) and produces s output frames x Cout channels, i.e. the
folded output IS the channel-last activation at the higher rate.  Crop (padding),
bias and PReLU are fused into the pass that writes the next layer's padded input.
Backward-data is a strided forward-convolution view of the output gradient; the
weight gradient is the same TN GEMM the encoder uses.
"""
import torch

from . import gemm, ops
from . import functional as Fn


def _cdiv(a, b):
    return -(-a // b)


class _LayerGeom(object):
    def __init__(self, Cin, Cout, k, s, pad, T_in):
        self.Cin, self.Cout, self.k, self.s, self.pad, self.T_in = Cin, Cout, k, s, pad, T_in
        self.taps = _cdiv(k, s)
        self.U = T_in + self.taps - 1                 # valid GEMM rows per sample
        self.Pd = T_in + 2 * (self.taps - 1)          # zero-padded input rows per sample
        self.L = (T_in - 1) * s - 2 * pad + k         # cropped output length


class DecoderPlan(object):
    def __init__(self, layers, B, T, device):
        self.B, self.T = B, T
        f32 = dict(dtype=torch.float32, device=device)
        self.geoms, Tin = [], T
        for (Cin, Cout, k, s, pad) in layers:
            g = _LayerGeom(Cin, Cout, k, s, pad, Tin)
            self.geoms.append(g)
            Tin = g.L
        self.xz, self.yfull, self.dyfull, self.Wu, self.dWu, self.Wb, self.dx = \
            [], [], [], [], [], [], []
        for g in self.geoms:
            self.xz.append(torch.zeros(B * g.Pd * g.Cin + g.taps * g.Cin + 64, **f32))
            self.yfull.append(torch.empty(B * g.U * g.s * g.Cout, **f32))
            self.dyfull.append(torch.zeros(B * g.U * g.s * g.Cout + g.k * g.Cout + 64, **f32))
            self.Wu.append(torch.empty(g.s * g.Cout * g.taps * g.Cin, **f32))
            self.dWu.append(torch.empty(g.s * g.Cout * g.taps * g.Cin, **f32))
            self.Wb.append(torch.empty(g.Cin * g.k * g.Cout, **f32))
            self.dx.append(torch.empty(B * g.T_in * g.Cin, **f32))
        cmax = max(g.Cout for g in self.geoms)
        self.ones = torch.ones(cmax, **f32)
        self.zeros = torch.zeros(cmax, **f32)
        self.acc = torch.zeros(4 * cmax, dtype=torch.float64, device=device)
        self.generation = 0


class _DecoderStackFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rows, plan, nlayers, *params):
        call = ops.call
        B, T = plan.B, plan.T
        rows = rows.detach().contiguous()
        plan.generation += 1
        G = plan.geoms
        p = Fn.gemm_precision()
        g0 = G[0]
        plan.xz[0][:B * g0.Pd * g0.Cin].view(B, g0.Pd, g0.Cin)[:, g0.taps - 1:g0.taps - 1 + T] \
            .copy_(rows.view(B, T, g0.Cin))
        out = None
        for i, g in enumerate(G):
            W, b, alpha = params[3 * i].detach(), params[3 * i + 1].detach(), \
                params[3 * i + 2].detach()
            call("pase_deconv_w_to_fwd", W.reshape(-1), plan.Wu[i], g.Cin, g.Cout, g.k, g.s, g.taps)
            gemm.nt(p, plan.xz[i], g.Cin, plan.xz[i].numel(), plan.Wu[i], g.taps * g.Cin,
                    plan.yfull[i], g.s * g.Cout, B * g.Pd, g.s * g.Cout, g.taps * g.Cin,
                    bias=b.repeat(g.s).contiguous(), rows_in=g.Pd, t_valid=g.U, rows_out=g.U)
            if i + 1 < len(G):
                nx = G[i + 1]
                dst, d_ss = plan.xz[i + 1][(nx.taps - 1) * nx.Cin:], nx.Pd * nx.Cin
            else:
                out = torch.empty(B * g.L, g.Cout, dtype=torch.float32, device=rows.device)
                dst, d_ss = out.reshape(-1), g.L * g.Cout
            C = g.Cout
            call("pase_bn_prelu_pad_fwd", plan.yfull[i][g.pad * C:], 0, g.U * g.s * C, B, g.L, C,
                 plan.ones[:C], plan.zeros[:C], alpha.reshape(-1), dst, None, 0, d_ss, C, 0, 0,
                 None, 0, 0, 0, 0)
        ctx.plan, ctx.generation = plan, plan.generation
        ctx.save_for_backward(*params)
        return out

    @staticmethod
    def backward(ctx, dh):
        call = ops.call
        plan = ctx.plan
        if plan.generation != ctx.generation:
            raise RuntimeError("pase_b200: decoder activations were overwritten by a later "
                               "forward before this backward ran")
        params = ctx.saved_tensors
        B, G = plan.B, plan.geoms
        p = Fn.gemm_precision()
        grads = [None] * len(params)
        src = dh.contiguous().reshape(-1)
        dev = dh.device
        for i in range(len(G) - 1, -1, -1):
            g, C = G[i], G[i].Cout
            W, b, alpha = params[3 * i].detach(), params[3 * i + 1].detach(), \
                params[3 * i + 2].detach()
            acc = plan.acc
            acc.zero_()
            S1, S2, dal, dbi = acc[:C], acc[C:2 * C], acc[2 * C:3 * C], acc[3 * C:4 * C]
            call("pase_bn_prelu_bwd_reduce", plan.yfull[i][g.pad * C:], 0, g.U * g.s * C, B, g.L, C,
                 plan.zeros[:C], plan.ones[:C], plan.ones[:C], plan.zeros[:C], alpha.reshape(-1),
                 src, 0, g.L * C, C, 0, 0, None, 0, 0, 0, None, 0, 0, 0, 0,
                 plan.dyfull[i][g.pad * C:], g.U * g.s * C, S1, S2, dal, None)
            # no normalisation in GDeconv1DBlock (mean 0, invstd 1): S1 = sum of du over every
            # kept position IS the bias gradient -- no separate column-sum pass over dY
            small = torch.empty(4 * C, dtype=torch.float32, device=dev)
            call("pase_cast_d2f", acc, small, 4 * C, 1.0)
            grads[3 * i + 2] = small[2 * C:3 * C].clone().view_as(alpha)
            grads[3 * i + 1] = small[:C].clone()
            # dY feeds the weight-gradient and the input-gradient GEMM: when both take the
            # tensor cores, one operand conversion
            dy, n_dy = plan.dyfull[i], plan.dyfull[i].numel()
            dyop = None
            if gemm.tn_ok(p, g.s * C, g.Cin, g.s * C, g.taps * g.Cin) and \
                    gemm.nt_ok(p, g.s * C, g.k * C, g.k * C):
                dyop = gemm.to_operand(p, dy, n_dy, "grad")
            gemm.tn(p, dy, g.s * C, n_dy, plan.xz[i], g.Cin, plan.xz[i].numel(), plan.dWu[i],
                    g.taps * g.Cin, g.s * C, g.taps * g.Cin, g.U, groups=B, pitchA=g.U, offA=0,
                    pitchB=g.Pd, a_op=dyop)
            dW = torch.empty_like(W)
            call("pase_deconv_w_from_fwd", plan.dWu[i], dW.reshape(-1), g.Cin, g.Cout, g.k, g.s,
                 g.taps)
            grads[3 * i] = dW
            if i > 0 or ctx.needs_input_grad[0]:
                call("pase_deconv_w_to_bwd", W.reshape(-1), plan.Wb[i], g.Cin, g.Cout, g.k)
                gemm.nt(p, dy, g.s * C, n_dy, plan.Wb[i], g.k * C, plan.dx[i], g.Cin, B * g.U,
                        g.Cin, g.k * C, rows_in=g.U, t_valid=g.T_in, rows_out=g.T_in,
                        a_kind="grad", a_op=dyop)
                src = plan.dx[i]
        dx = None
        if ctx.needs_input_grad[0]:
            dx = plan.dx[0].view(B * G[0].T_in, G[0].Cin).clone()
        return (dx, None, None) + tuple(grads)


def decoder_stack(minion, rows, B, T):
    """Runs the minion's leading GDeconv blocks on (B*T, C) rows.  Returns
    ((B*L, C_last) rows, L)."""
    layers, params = [], []
    for blk in minion.blocks[:minion.n_deconv]:
        W = blk.deconv.weight
        layers.append((W.shape[0], W.shape[1], blk.kwidth, blk.stride, blk.pad))
        params += [W, blk.deconv.bias, blk.act.weight]
    key = (B, T, str(rows.device))
    plan = minion._plans.get(key)
    if plan is None:
        if len(minion._plans) >= 2:
            minion._plans.clear()
        plan = DecoderPlan(layers, B, T, rows.device)
        minion._plans[key] = plan
    out = _DecoderStackFn.apply(rows, plan, len(layers), *params)
    return out, plan.geoms[-1].L
