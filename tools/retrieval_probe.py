"""Times full-corpus VCMR / VR / SVMR ranking at the TVR eval config on one GPU: the native path
(evalpass.rank_modularized on csrc/rank.cu) against a torch restatement of the reference's
eval_vcmr.py:232-323 plus its host-side SVMR (:326-354), on the same synthetic corpus and queries.

    python tools/retrieval_probe.py [--clips 2000] [--queries 10000] [--out result.json]

Corpus: seeded, `--clips` clips of 40..100 frames (L = 100), H = 768, zeros at padded frames as
embed_video_corpus leaves them. Queries in batches of 80, K = 100 clips, N = 200 moments, span band
[2, 16), width-5 span convolutions. Per-batch times are CUDA-event means over `--iters` batches after
a warm-up; the full pass ranks `--queries` queries batch by batch including each batch's
device->host copy (and, for the torch path, the host SVMR at the end), timed to a device
synchronise. The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hero_b200 import evalpass  # noqa: E402

B, K, N, MIN_L, MAX_L, ALPHA, H, L = 80, 100, 200, 2, 16, 20.0, 768, 100


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        return name, r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return name, "unknown"


def make_inputs(n_clips, n_queries, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lens = torch.randint(40, L + 1, (n_clips,), device="cuda", generator=g)
    lens[0] = L
    mask = (torch.arange(L, device="cuda")[None] < lens[:, None])
    frames = torch.randn(n_clips, L, H, device="cuda", generator=g) * mask[..., None]
    m = torch.randn(n_queries, H, device="cuda", generator=g)
    lin = torch.nn.Linear(H, H).cuda()
    with torch.no_grad():
        lin.weight.copy_(torch.randn(H, H, device="cuda", generator=g) * 0.02)
        lin.bias.zero_()
        p = lin(m)
    w = torch.randn(2, 5, device="cuda", generator=g) * 0.3
    gt = torch.randint(0, n_clips, (n_queries,), device="cuda", generator=g)
    return frames, mask, m, p, w, gt


def generate_min_max_length_mask(shape, min_l, max_l):
    """Band mask of the span (start, end) matrix, as the reference's tvr_eval_utils builds it."""
    ones = np.ones((1,) * (len(shape) - 2) + tuple(shape[-2:]), dtype=np.float32)
    return np.triu(ones, k=min_l) * (1 - np.triu(ones, k=max_l))


class TorchPath:
    """eval_vcmr.py:232-323 restated in torch (cross span logits for every clip, (Nq, K, L, L)
    products, full sort) + the host SVMR of :326-354."""

    def __init__(self, frames, mask, w):
        self.frames, self.maskf = frames, mask.float()
        conv = dict(in_channels=1, out_channels=1, kernel_size=5, padding=2, bias=False)
        self.st_conv, self.ed_conv = torch.nn.Conv1d(**conv).cuda(), torch.nn.Conv1d(**conv).cuda()
        with torch.no_grad():
            self.st_conv.weight.copy_(w[0].view(1, 1, 5))
            self.ed_conv.weight.copy_(w[1].view(1, 1, 5))
        self.svmr_st, self.svmr_ed = [], []

    @torch.no_grad()
    def batch(self, m, p, gt):
        nq = m.shape[0]
        nv = self.frames.shape[0]
        # video scores (model/pretrain.py:364-413)
        qn = F.normalize(m, dim=-1, eps=1e-5)
        cn = F.normalize(self.frames, dim=-1, eps=1e-5)
        s = torch.einsum("md,nld->mln", qn, cn)
        mk = self.maskf.t()[None]
        s = (s * mk + (1 - mk) * -1e4).max(1).values
        # span logits for every (query, clip) pair (cross=True)
        sim = torch.einsum("md,nld->mnl", p, self.frames).reshape(nq * nv, 1, L)
        st = self.st_conv(sim).view(nq, nv, L)
        ed = self.ed_conv(sim).view(nq, nv, L)
        mm = self.maskf[None]
        st = F.softmax(st * mm + (1 - mm) * -1e4, dim=-1)
        ed = F.softmax(ed * mm + (1 - mm) * -1e4, dim=-1)
        rows = torch.arange(nq, device=m.device)
        self.svmr_st.append(st[rows, gt].float().cpu().numpy())
        self.svmr_ed.append(ed[rows, gt].float().cpu().numpy())
        f = torch.exp(ALPHA * s)
        vs, vi = torch.topk(f, K, dim=1, largest=True)
        vr = (vs.cpu().numpy(), vi.cpu().numpy())
        r = rows.unsqueeze(1)
        prod = torch.einsum("qvm,qv,qvn->qvmn", st[r, vi], vs, ed[r, vi])
        band = generate_min_max_length_mask(prod.shape, MIN_L, MAX_L)
        prod *= torch.from_numpy(band).to(prod.device)
        ss, si = torch.sort(prod.reshape(nq, -1), dim=1, descending=True)
        return vr, (si[:, :N].cpu().numpy(), ss[:, :N].cpu().numpy())

    def host_svmr(self):
        st, ed = np.concatenate(self.svmr_st), np.concatenate(self.svmr_ed)
        prod = np.einsum("bm,bn->bmn", st, ed)
        prod *= generate_min_max_length_mask(prod.shape, MIN_L, MAX_L)
        out = []
        for e in prod:
            order = np.argsort(e, axis=None)[::-1][:N]
            r, c = np.unravel_index(order, e.shape)
            out.append(np.stack([r, c, e[r, c]], 1))
        self.svmr_st, self.svmr_ed = [], []
        return out


def ours_batch(corpus, m, p, w, gt):
    out = evalpass.rank_modularized(corpus, m, p, w[0], w[1], q2c_alpha=ALPHA, max_video=K,
                                    min_pred_l=MIN_L, max_pred_l=MAX_L, max_before_nms=N,
                                    gt_vidx=gt)
    return evalpass._to_host(out)


def per_batch_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn(0)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(iters):
        fn(i)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2000)
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("retrieval_probe needs a CUDA device")
    name, power = card()
    frames, mask, m, p, w, gt = make_inputs(a.clips, a.queries)
    corpus = evalpass.VideoCorpus(frames, mask)
    tp = TorchPath(frames, mask, w)
    n_b = (a.queries + B - 1) // B

    def sl(i):
        i %= n_b
        return slice(i * B, min(a.queries, (i + 1) * B))

    # agreement on one batch: VR lists and the VCMR top scores
    (ov, oi), = [ours_batch(corpus, m[sl(0)], p[sl(0)], w, gt[sl(0)])["VR"]]
    (tv, ti), (tsi, tss) = tp.batch(m[sl(0)], p[sl(0)], gt[sl(0)])
    tp.svmr_st, tp.svmr_ed = [], []
    oc = ours_batch(corpus, m[sl(0)], p[sl(0)], w, gt[sl(0)])["VCMR"][0]
    agree = dict(vr_index_match=float((oi == ti).mean()),
                 vr_rel_err=float(np.abs(ov - tv).max() / np.abs(tv).max()),
                 vcmr_rel_err=float(np.abs(oc - tss).max() / np.abs(tss).max()))

    ours_ms = per_batch_ms(lambda i: ours_batch(corpus, m[sl(i)], p[sl(i)], w, gt[sl(i)]),
                           a.iters)
    torch_ms = per_batch_ms(lambda i: tp.batch(m[sl(i)], p[sl(i)], gt[sl(i)]), a.iters)
    tp.svmr_st, tp.svmr_ed = [], []

    torch.cuda.synchronize()
    t = time.perf_counter()
    for i in range(n_b):
        ours_batch(corpus, m[sl(i)], p[sl(i)], w, gt[sl(i)])
    torch.cuda.synchronize()
    ours_full = time.perf_counter() - t
    t = time.perf_counter()
    for i in range(n_b):
        tp.batch(m[sl(i)], p[sl(i)], gt[sl(i)])
    torch.cuda.synchronize()
    t_dev = time.perf_counter() - t
    tp.host_svmr()
    torch_full = time.perf_counter() - t
    res = dict(card=name, power_limit_and_max_sm_clock=power, clips=a.clips, queries=a.queries,
               batch=B, K=K, N=N, band=[MIN_L, MAX_L],
               ours_ms_per_batch=round(ours_ms, 3), torch_ms_per_batch=round(torch_ms, 3),
               ours_full_pass_s=round(ours_full, 3), torch_full_pass_s=round(torch_full, 3),
               torch_full_pass_device_loop_s=round(t_dev, 3), agreement=agree)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
