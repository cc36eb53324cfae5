"""``pase_adam_flat``: one optimizer step per row of the segment table, by its algorithm column
(0 Adam, 1 RAdam).  RAdam restates the reference's RAdam (pase/models/WorkerScheduler/radam.py:
21-76) from the table's fp32 hyper-parameters, with rho and the step size in float64 as the
kernel computes them."""
import math
import struct

import torch

ROW = "<qqffffffq"


def radam_constants(lr, beta1, beta2, weight_decay, t):
    """(rectified, step_size, -(weight_decay * lr)) of step t, in float64."""
    b2t = beta2 ** t
    rho_inf = 2.0 / (1.0 - beta2) - 1.0
    rho = rho_inf - 2.0 * t * b2t / (1.0 - b2t)
    bias1 = 1.0 - beta1 ** t
    if rho >= 5.0:
        step = lr * math.sqrt((1.0 - b2t) * (rho - 4.0) / (rho_inf - 4.0) * (rho - 2.0) / rho *
                              rho_inf / (rho_inf - 2.0)) / bias1
        return True, step, -(weight_decay * lr)
    return False, lr / bias1, -(weight_decay * lr)


def pase_adam_flat(param, grad, exp_avg, exp_avg_sq, n, seg_table, nseg, steps, grad_scale):
    raw = seg_table[:nseg * 6].numpy().tobytes()
    for i in range(nseg):
        a, b, lr, b1, b2, eps, wd, algo, si = struct.unpack_from(ROW, raw, i * 48)
        t = float(steps[si])
        if algo == 0.0:
            # torch.optim.Adam (amsgrad / maximize off, L2 weight decay)
            g = grad[a:b] * grad_scale + wd * param[a:b]
            exp_avg[a:b] = b1 * exp_avg[a:b] + (1 - b1) * g
            exp_avg_sq[a:b] = b2 * exp_avg_sq[a:b] + (1 - b2) * g * g
            bias1, bias2 = 1 - b1 ** t, 1 - b2 ** t
            denom = exp_avg_sq[a:b].sqrt() / math.sqrt(bias2) + eps
            param[a:b] -= (lr / bias1) * exp_avg[a:b] / denom
            continue
        assert algo == 1.0, algo
        rect, step, decay = radam_constants(lr, b1, b2, wd, t)
        step, decay = float(torch.tensor(step, dtype=torch.float32)), float(
            torch.tensor(decay, dtype=torch.float32))
        g = grad[a:b] * grad_scale
        m, v, p = exp_avg[a:b], exp_avg_sq[a:b], param[a:b]
        m.copy_(b1 * m + (1 - b1) * g)
        v.copy_(b2 * v + (1 - b2) * g * g)
        p.add_(decay * p)
        if rect:
            p.add_(-step * (m / (v.sqrt() + eps)))
        else:
            p.add_(-step * m)
