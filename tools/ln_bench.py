"""Device-time micro-benchmark of the row kernels at bench shapes (CUDA events, buffers rotated
through > L2 so every launch reads HBM; kernels shorter than ~10 us are host-launch bound here).
Usage: python tools/ln_bench.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hero_b200 import ops

dev = torch.device("cuda:0")
H = 768
drop = ops.drop_params(0.1, 77)


def timeit(fn, n=40):
    for i in range(4):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


for M in (16512, 3200):
    R = 12 if M > 10000 else 40           # rotate through R buffer sets (> 50 MB of L2)
    xs = [torch.randn(M, H, device=dev).bfloat16() for _ in range(R)]
    dys = [torch.randn(M, H, device=dev).bfloat16() for _ in range(R)]
    ys = [torch.empty(M, H, dtype=torch.bfloat16, device=dev) for _ in range(R)]
    dxs = [torch.empty(M, H, dtype=torch.bfloat16, device=dev) for _ in range(R)]
    dxd = [torch.empty(M, H, dtype=torch.bfloat16, device=dev) for _ in range(R)]
    g, b = torch.ones(H, device=dev), torch.zeros(H, device=dev)
    mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
    dg, db, dbias = (torch.zeros(H, device=dev) for _ in range(3))
    ops.ln_fwd(xs[0], g, b, 1e-12, ys[0], n_rows=M, mean=mean, rstd=rstd)
    t_f = timeit(lambda i: ops.ln_fwd(xs[i % R], g, b, 1e-12, ys[i % R], n_rows=M, mean=mean,
                                      rstd=rstd))
    t_b = timeit(lambda i: ops.ln_bwd(dys[i % R], xs[i % R], g, mean, rstd, n_rows=M,
                                      dx=dxs[i % R], dx_drop=dxd[i % R], drop2=drop))
    t_p = timeit(lambda i: ops.ln_bwd(dys[i % R], xs[i % R], g, mean, rstd, n_rows=M,
                                      dx=dxs[i % R], dx_drop=dxd[i % R], drop2=drop, dgamma=dg,
                                      dbeta=db, dbias=dbias))
    t_c = timeit(lambda i: ops.colsum(dys[i % R], dbias))
    by = M * H * 2 / 1e6
    print(f"M={M}: ln_fwd {t_f:.1f} us ({2 * by / t_f:.2f} TB/s)  ln_bwd rows {t_b:.1f} us "
          f"({4 * by / t_b:.2f} TB/s)  rows+params {t_p:.1f} us  colsum {t_c:.1f} us "
          f"({by / t_c:.2f} TB/s)")

    # fp32 pre-LayerNorm sums (the residual stream of the transformer layers)
    xs32 = [x.float() for x in xs[:6]]
    y32 = torch.empty(M, H, device=dev)
    R2 = len(xs32)
    t_f = timeit(lambda i: ops.ln_fwd(xs32[i % R2], g, b, 1e-12, ys[i % R], n_rows=M, mean=mean,
                                      rstd=rstd))
    t_f2 = timeit(lambda i: ops.ln_fwd(xs32[i % R2], g, b, 1e-12, ys[i % R], n_rows=M, mean=mean,
                                       rstd=rstd, y_f32=y32))
    t_p = timeit(lambda i: ops.ln_bwd(dys[i % R], xs32[i % R2], g, mean, rstd, n_rows=M,
                                      dx=dxs[i % R], dx_drop=dxd[i % R], drop2=drop, dgamma=dg,
                                      dbeta=db, dbias=dbias))
    print(f"M={M} fp32 rows: ln_fwd {t_f:.1f} us ({3 * by / t_f:.2f} TB/s)  +fp32 copy {t_f2:.1f} us "
          f"({5 * by / t_f2:.2f} TB/s)  ln_bwd rows+params {t_p:.1f} us ({5 * by / t_p:.2f} TB/s)")

# 4352-wide rows: the video-feature LayerNorm of ImageEmbeddings (model/embed.py:108-116), fp32
# features in, bf16 normalised rows out (+ the bf16 low halves for the split GEMM when asked)
D, M = 4352, 3200
R = 4
xw = [torch.randn(M, D, device=dev) for _ in range(R)]
yw = [torch.empty(M, D, dtype=torch.bfloat16, device=dev) for _ in range(R)]
gw, bw = torch.ones(D, device=dev), torch.zeros(D, device=dev)
mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
t_w = timeit(lambda i: ops.ln_fwd(xw[i % R], gw, bw, 1e-12, yw[i % R], n_rows=M, mean=mean, rstd=rstd))
print(f"wide rows {M} x {D} fp32 -> bf16: ln_fwd {t_w:.1f} us ({M * D * 6 / 1e6 / t_w:.2f} TB/s)")
