"""Times the GEMM variants that have a wide (128 x 256) form at the training step's shapes, with
both tilings side by side and the tiling / split count the auto chooser picks (CUDA events around
single launches, L2 flushed between reps). Data for fitting the chooser's cost model in
csrc/gemm_wgmma.cu. Prints one line per shape and writes every timing as JSON to --out.

    python tools/gemm_probe.py [--tokens 16512,3200] [--max-split 8] [--out gemm_probe.json]
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from hero_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
H, I = 768, 3072


def timeit(fn, reps=15):
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
    return ts[len(ts) // 2]


def auto_choice(fn):
    """(block_n, ms) of one profiled launch with block_n = 0, from the per-launch dump."""
    path = os.path.join(tempfile.mkdtemp(), "gemm.csv")
    os.environ["HERO_GEMM_PROFILE_DUMP"] = path
    ops.start_gemm_profile()
    fn()
    ops.stop_gemm_profile()
    del os.environ["HERO_GEMM_PROFILE_DUMP"]
    with open(path) as f:
        row = f.read().splitlines()[1].split(",")
    return int(row[7])


def rnd(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device=dev) * scale).to(dtype)


def cases(m):
    """(name, m, n, k, call(block_n, k_splits)) for the wide-capable GEMMs of one layer at m tokens."""
    out = []
    # forward into the fp32 residual stream: LayerNorm-form residual + dropout
    for name, k in (("ffn_down_fwd", I), ("out_proj_fwd", H)):
        a, w = rnd(m, k), rnd(H, k, scale=0.02)
        bias, pre = torch.randn(H, device=dev), torch.randn(m, H, device=dev)
        ln = (pre.mean(-1), torch.rsqrt(pre.var(-1, unbiased=False) + 1e-12),
              torch.ones(H, device=dev), torch.zeros(H, device=dev))
        o = torch.empty(m, H, device=dev)
        out.append((name, m, H, k, lambda bn, sp, a=a, w=w, bias=bias, pre=pre, ln=ln, o=o: ops.gemm(
            a, w, o, bias=bias, resid=pre, resid_ln=ln, drop=ops.drop_params(0.1, 1), block_n=bn)))
    # dgrads with a bf16 residual, B MN-major
    for name, k in (("ffn_up_dgrad_da", I), ("qkv_dgrad_dx", 3 * H)):
        dy, w, r = rnd(m, k), rnd(k, H, scale=0.05), rnd(m, H)
        o = torch.empty(m, H, dtype=torch.bfloat16, device=dev)
        out.append((name, m, H, k, lambda bn, sp, dy=dy, w=w, r=r, o=o: ops.gemm(
            dy, w, o, b_mn=True, resid=r, block_n=bn)))
    # weight gradients, split-K fp32 atomics (layout (1,1)); 4352: the embedding projection
    wg = [("dW2", H, I), ("dW1", I, H), ("dWqkv", 3 * H, H), ("dWo", H, H)]
    if m != 16512:
        wg.append(("dWproj", H, 4352))
    for name, n_out, k_in in wg:
        dy, x = rnd(m, n_out, scale=0.1), rnd(m, k_in)
        o = torch.zeros(n_out, k_in, device=dev)
        out.append(("wgrad_" + name, n_out, k_in, m, lambda bn, sp, dy=dy, x=x, o=o: ops.gemm(
            dy, x, o, a_mn=True, b_mn=True, accumulate_f32=True, k_splits=sp, block_n=bn)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="16512,3200")
    ap.add_argument("--max-split", type=int, default=8)
    ap.add_argument("--out", default="gemm_probe.json", help="JSON file for all timings")
    args = ap.parse_args()
    res = []
    for m in (int(t) for t in args.tokens.split(",")):
        for name, gm, gn, gk, call in cases(m):
            splits = range(1, args.max_split + 1) if name.startswith("wgrad") else (0,)
            row = dict(name=name, tokens=m, m=gm, n=gn, k=gk, ms={})
            for sp in splits:
                for bn in (128, 256):
                    row["ms"][f"{bn}/{sp}"] = timeit(lambda: call(bn, sp))
            row["auto_ms"] = timeit(lambda: call(0, 0))
            row["auto_block_n"] = auto_choice(lambda: call(0, 0))
            fl = 2.0 * gm * gn * gk
            best = min(row["ms"], key=row["ms"].get)
            print(f"{name:16s} tokens {m:5d} {gm}x{gn}x{gk}  auto bn{row['auto_block_n']} "
                  f"{row['auto_ms']:.3f} ms ({fl / row['auto_ms'] / 1e9:.0f} TF/s)  best {best} "
                  f"{row['ms'][best]:.3f}  | " +
                  " ".join(f"{key}:{v:.3f}" for key, v in row["ms"].items()), flush=True)
            res.append(row)
    with open(args.out, "w") as f:
        json.dump(dict(device=torch.cuda.get_device_name(0), results=res), f, indent=1)


if __name__ == "__main__":
    main()
