"""Attention / LayerNorm launches at bench shapes for `ncu --set full`."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from hero_b200 import ops
from hero_b200.plan import DeviceIndex, SeqPlan

dev = torch.device("cuda:0")
heads, H = 12, 768
lens = [25] * 640 + [16] * 32
mask = np.zeros((len(lens), 25), np.int64)
for r, n in enumerate(lens):
    mask[r, :n] = 1
sp = SeqPlan(mask)
att = sp.attn(DeviceIndex(sp.arrays("s_"), dev), "s_")
M = sp.n_tok
qkv = torch.randn(M, 3 * H, device=dev).bfloat16()
ctx = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
lse = torch.empty(M, heads, device=dev)
dctx = torch.randn(M, H, device=dev).bfloat16()
dqkv = torch.empty_like(qkv)
drop = ops.drop_params(0.1, 77)
x = torch.randn(M, H, device=dev).bfloat16()
g, b = torch.ones(H, device=dev), torch.zeros(H, device=dev)
y = torch.empty_like(x)
mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
dx, dxd = torch.empty_like(x), torch.empty_like(x)
dg, db, dbias = torch.zeros(H, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev)
for _ in range(3):
    ops.attn_fwd(qkv, att, ctx, heads=heads, drop=drop, lse=lse)
    ops.attn_bwd(qkv, att, ctx, dctx, lse, dqkv, heads=heads, drop=drop)
    ops.ln_fwd(x, g, b, 1e-12, y, n_rows=M, mean=mean, rstd=rstd)
    ops.ln_bwd(dctx, x, g, mean, rstd, n_rows=M, dx=dx, dx_drop=dxd, drop2=drop, dgamma=dg, dbeta=db)
torch.cuda.synchronize()
print("done")
