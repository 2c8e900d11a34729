"""Times the wgmma GEMM on the encoder's shapes (CUDA events, L2 flushed between reps)."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hero_b200 import ops

dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        s, e = torch.cuda.Event(True), torch.cuda.Event(True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    res = []
    shapes = [("qkv", 16000, 2304, 768), ("out", 16000, 768, 768), ("ffn1", 16000, 3072, 768),
              ("ffn2", 16000, 768, 3072), ("c_ffn1", 3200, 3072, 768), ("proj", 3200, 768, 4352),
              ("big", 8192, 8192, 8192)]
    for name, m, n, k in shapes:
        a = torch.randn(m, k, device=dev).bfloat16()
        w = (torch.randn(n, k, device=dev) * 0.05).bfloat16()
        bias = torch.randn(n, device=dev)
        out = torch.empty(m, n, dtype=torch.bfloat16, device=dev)
        for bn, pair in ((128, 1), (256, 1), (256, 2)):
            for act in (ops.ACT_NONE, ops.ACT_GELU):
                med, best = timeit(lambda: ops.gemm(a, w, out, bias=bias, act=act, block_n=bn,
                                                    cta_pair=pair))
                tf = 2.0 * m * n * k / (med * 1e-3) / 1e12
                res.append(dict(kind="fwd", name=name, m=m, n=n, k=k, block_n=bn * (pair == 2 and 10 or 1), act=act,
                                ms=med, best_ms=best, tflops=tf))
                print(res[-1], flush=True)
        med, best = timeit(lambda: torch.matmul(a, w.t()))
        print(dict(kind="torch.matmul", name=name, ms=med, tflops=2.0 * m * n * k / (med * 1e-3) / 1e12), flush=True)
        # dgrad: dX[m,k] = dY[m,n] @ W[n,k]
        dy = torch.randn(m, n, device=dev).bfloat16()
        dx = torch.empty(m, k, dtype=torch.bfloat16, device=dev)
        if k % 64 == 0:
            for pair in (1, 2):
                med, best = timeit(lambda: ops.gemm(dy, w, dx, b_mn=True, cta_pair=pair))
                print(dict(kind="dgrad pair%d" % pair, name=name, ms=med, tflops=2.0 * m * n * k / (med * 1e-3) / 1e12), flush=True)
        # wgrad: dW[n,k] += dY^T X
        if m % 64 == 0 or True:
            dw = torch.zeros(n, k, device=dev)
            mm = (m // 64) * 64
            try:
                for pair in (1, 2):
                    med, best = timeit(lambda: ops.gemm(dy[:mm], a[:mm], dw, a_mn=True, b_mn=True, accumulate_f32=True, cta_pair=pair))
                    print(dict(kind="wgrad pair%d" % pair, name=name, ms=med, tflops=2.0 * mm * n * k / (med * 1e-3) / 1e12), flush=True)
            except Exception as ex:
                print("wgrad failed", name, ex)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open("gpurun_out/gemm_probe.json", "w"))


if __name__ == "__main__":
    main()
