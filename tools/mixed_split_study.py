#!/usr/bin/env python
"""CPU study for a GEMM precision scheme: keep the main product in TF32 and do the two
error-compensation products of 3xTF32 in bf16 (twice the tensor rate), i.e.

    D = trunc_tf32(a) * rn_tf32(b)                       (tf32 pass, as today)
      + bf16(a - trunc_tf32(a)) * bf16(b)                (bf16 pass)
      + bf16(a) * bf16(b - rn_tf32(b))                   (bf16 pass)

and, cheaper still, three bf16 products of a two-term bf16 split of both operands
(a1*b1 + a1*b2 + a2*b1: 1.5 TF32-pass equivalents of tensor time against 3 today, and bf16
operand pairs instead of fp32 + residual, i.e. half the operand bytes), and compare their
errors against fp64 with today's 3xTF32 and with single-pass TF32, on operands
shaped like the PASE+ layers (zero-mean activations, K up to 5632).  Products are exact in
fp32 for 8-/11-bit mantissas, accumulation is emulated in fp64 (the kernels fold K = 128
chunks into fp32 sums; that part is common to all schemes).
"""
import torch


def trunc_tf32(x):
    return (x.contiguous().view(torch.int32) & -8192).view(torch.float32)


def rn_tf32(x):
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    u = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    u = torch.where(u >= 2 ** 31, u - 2 ** 32, u)
    return u.to(torch.int32).view(torch.float32)


def bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


def study(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g) * torch.rand(1, K, generator=g)     # uneven channel scales
    b = torch.randn(N, K, generator=g) / K ** 0.5
    ref = a.double() @ b.double().t()
    ah, bh = trunc_tf32(a), rn_tf32(b)
    al, bl = rn_tf32(a - ah), rn_tf32(b - bh)
    d = lambda x, y: x.double() @ y.double().t()
    one = d(ah, bh)
    three = one + d(al, bh) + d(ah, bl)
    mixed = one + d(bf16(a - ah), bf16(b)) + d(bf16(a), bf16(b - bh))
    a1, b1 = bf16(a), bf16(b)
    a2, b2 = bf16(a - a1), bf16(b - b1)
    b3 = d(a1, b1) + d(a1, b2) + d(a2, b1)
    scale = ref.abs().max()
    out = {}
    for name, v in (("tf32", one), ("3xtf32", three), ("tf32+2bf16", mixed),
                    ("3xbf16 (2-term split)", b3)):
        e = (v - ref).abs()
        out[name] = (float(e.max() / scale), float((e.pow(2).sum() / ref.pow(2).sum()).sqrt()))
    return out


if __name__ == "__main__":
    print("| M x N x K | scheme | max err / max|ref| | rel. L2 |")
    print("|---|---|---:|---:|")
    for (M, N, K) in ((512, 256, 704), (512, 256, 2816), (256, 512, 5632), (512, 1536, 1024)):
        r = study(M, N, K, 7 + K)
        for name, (mx, l2) in r.items():
            print("| %d x %d x %d | %s | %.2e | %.2e |" % (M, N, K, name, mx, l2))
