"""Encoder-shaped GEMM launches for `ncu --set full --import-source on`:
the five epilogue families at the cross-modal (M = 16512) and temporal (M = 3200) token counts."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from hero_b200 import ops

dev = torch.device("cuda:0")
REPS = int(os.environ.get("REPS", "1"))


def bf(*shape, s=1.0):
    return (torch.randn(*shape, device=dev) * s).bfloat16()


for M in (16512, 3200):
    x = bf(M, 768)
    w1, b1 = bf(3072, 768, s=0.05), torch.randn(3072, device=dev)
    wq, bq = bf(2304, 768, s=0.05), torch.randn(2304, device=dev)
    wo, bo = bf(768, 768, s=0.05), torch.randn(768, device=dev)
    w2, b2 = bf(768, 3072, s=0.05), torch.randn(768, device=dev)
    f, pre = torch.empty(M, 3072, dtype=torch.bfloat16, device=dev), torch.empty(M, 3072, dtype=torch.bfloat16, device=dev)
    qkv = torch.empty(M, 2304, dtype=torch.bfloat16, device=dev)
    h32 = torch.randn(M, 768, device=dev)
    s1 = torch.empty(M, 768, device=dev)
    dw = torch.zeros(3072, 768, device=dev)
    dx = torch.empty(M, 768, dtype=torch.bfloat16, device=dev)
    drop = ops.drop_params(0.1, 99)
    for _ in range(REPS):
        ops.gemm(x, wq, qkv, bias=bq)                                   # fused QKV
        ops.gemm(x, wo, s1, bias=bo, resid=h32, drop=drop)              # out-proj: fp32 residual stream
        ops.gemm(x, w1, f, bias=b1, act=ops.ACT_GELU, aux_out=pre)      # FFN-up + erf-GELU (+GELU')
        ops.gemm(f, w2, s1, bias=b2, resid=h32, drop=drop)              # FFN-down: fp32 residual stream
        ops.gemm(x, w2, f, b_mn=True, act=ops.ACT_GELU_GRAD, aux_in=pre)  # dgrad * GELU' (N = 3072)
        ops.gemm(f, w1, dx, b_mn=True, resid=x)                         # dgrad K = 3072 + residual
        ops.gemm(f, x, dw, a_mn=True, b_mn=True, accumulate_f32=True)   # wgrad (K = tokens)
torch.cuda.synchronize()
print("done")
