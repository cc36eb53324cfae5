"""GPU probe: does the tf32 tensor-core GEMM truncate or round its fp32 inputs?  (decides whether the
'hi' operand of the 3xTF32 scheme could be the original array).  Prints one line."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from pase_b200 import _lib
import emul

torch.manual_seed(0)
M = N = 128
K = 256
A, B = torch.randn(M * K + 64), torch.randn(N * K)
At = emul.core._tf32_trunc(A)
Bt = emul.core._tf32_trunc(B)
outs = []
for a, b in ((A, B), (At, Bt)):
    C = torch.zeros(M * N).cuda()
    _lib.call("pase_tc_gemm_nt", a.cuda(), None, (M * K + 64) // K, K, b.cuda(), None, K, C, N, M, N, K,
              1.0, None, None, M, M, M, 1, None, None, 0, 0, 0)
    outs.append(C.cpu())
ref_t = (At[:M * K].view(M, K).double() @ Bt.view(N, K).double().t()).float().reshape(-1)
ref_f = (A[:M * K].view(M, K).double() @ B.view(N, K).double().t()).float().reshape(-1)
print("tf32 probe: raw-vs-pretruncated max diff %.3e | raw err vs truncated-ref %.3e | raw err vs fp32-ref %.3e"
      % (float((outs[0] - outs[1]).abs().max()), float((outs[0] - ref_t).abs().max()),
         float((outs[0] - ref_f).abs().max())))
