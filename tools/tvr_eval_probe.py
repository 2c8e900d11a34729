"""Times the NMS-and-metrics half of full-corpus VCMR evaluation at the TVR eval config on one GPU:
the native path (evalpass.full_vcmr_eval, NMS on csrc/nms.cu, vectorised metrics) against
full_vcmr_predictions followed by a plain host restatement of the reference's post-processing
(greedy NMS with one IoU call per pair, per-query metric loop), on the same synthetic corpus and
queries, run back to back.

    python tools/tvr_eval_probe.py [--clips 2000] [--queries 10000] [--out result.json]

Corpus and queries are those of tools/retrieval_probe.py (seeded, 2 000 clips of 40..100 frames,
H = 768), ranked in batches of 80 with K = 100, N = max_before_nms = 200, max_after_nms = 100,
nms_thd = 0.5. The query encoder is bypassed: each batch ranks stored modularized queries, in both
paths. Reported: the NMS kernel's time per batch (VCMR and SVMR launches, CUDA events over
`--iters` batches after a warm-up), and wall time of the two full passes to the last metric. The
card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hero_b200 import evalpass  # noqa: E402
from tools.retrieval_probe import ALPHA, B, K, MAX_L, MIN_L, N, card, make_inputs  # noqa: E402

MAX_AFTER_NMS, NMS_THD, INTERVAL = 100, 0.5, 1.5


class _Stub(torch.nn.Module):
    lw_neg_ctx = lw_neg_q = 8


def _setup(n_clips, n_queries):
    frames, mask, m, p, w, gt = make_inputs(n_clips, n_queries)
    corpus = evalpass.VideoCorpus(frames, mask)
    video_ids = [f"clip{i:05d}" for i in range(n_clips)]
    video2idx = {v: i for i, v in enumerate(video_ids)}
    gt = gt.cpu().tolist()
    batches = []
    for a in range(0, n_queries, B):
        b = min(n_queries, a + B)
        batches.append(dict(qids=list(range(a, b)), vids=[video_ids[g] for g in gt[a:b]],
                            targets=torch.zeros(b - a, 2, dtype=torch.long),
                            query_input_ids=torch.arange(a, b)[:, None],
                            query_pos_ids=torch.zeros(1, 1, dtype=torch.long),
                            query_attn_masks=torch.ones(b - a, 1, dtype=torch.long)))
    rng = np.random.default_rng(0)
    ground_truth = []
    for q in range(n_queries):
        s = int(rng.integers(0, 80))
        ground_truth.append(dict(desc_id=q, desc="", type=("v", "t", "vt")[q % 3],
                                 vid_name=video_ids[gt[q]],
                                 ts=[s * INTERVAL, (s + int(rng.integers(2, 16))) * INTERVAL]))

    def rank_queries(model, corpus_, qb, *, tasks, gt_vidx=None, **kw):
        r = qb["query_input_ids"][:, 0].cuda(non_blocking=True)
        return evalpass.rank_modularized(corpus_, m[r], p[r], w[0], w[1], tasks=tasks,
                                         gt_vidx=gt_vidx, **kw)
    evalpass.rank_queries = rank_queries
    return corpus, batches, video_ids, video2idx, ground_truth, m, p, w


# ---- host restatement of the reference's post-processing (tvr_eval_utils / tvr_standalone_eval)
def _iou(a, b):
    inter = max(0, min(a[1], b[1]) - max(a[0], b[0]))
    union = max(a[1], b[1]) - min(a[0], b[0])
    return 0 if union == 0 else 1.0 * inter / union


def _greedy(preds, thd, cap=100):
    rest = sorted(preds, key=lambda x: x[2], reverse=True)
    kept = []
    while rest and len(kept) < cap:
        head = rest.pop(0)
        kept.append(head)
        rest = [x for x in rest if _iou(head, x) <= thd]
    return kept


def host_nms(sub, n_in):
    out = dict(video2idx=sub["video2idx"])
    out["SVMR"] = [dict(e, predictions=[[p[0][0]] + x for x in _greedy([q[1:] for q in p], NMS_THD)]
                        [:MAX_AFTER_NMS] if p else []) for e in sub["SVMR"]
                   for p in [e["predictions"][:n_in]]]
    vcmr = []
    for e in sub["VCMR"]:
        groups = defaultdict(list)
        for x in e["predictions"][:n_in]:
            groups[x[0]].append(x[1:])
        merged = [[v] + x for v, g in groups.items() for x in _greedy(g, NMS_THD)]
        vcmr.append(dict(e, predictions=sorted(merged, key=lambda x: x[3],
                                               reverse=True)[:MAX_AFTER_NMS]))
    out["VCMR"] = vcmr
    return out


def host_metrics(sub, ground_truth, thds=(0.5, 0.7)):
    """Per-query loop as eval_by_task_type runs it; returns the R@k means."""
    gt = {e["desc_id"]: e for e in ground_truth}
    res = {}
    for task in ("VCMR", "SVMR", "VR"):
        if task not in sub:
            continue
        hits = defaultdict(list)
        for e in sub[task]:
            g = gt[e["desc_id"]]
            pr = np.array([x[:3] for x in e["predictions"][:100]], dtype=np.float32).reshape(-1, 3)
            match = pr[:, 0] == sub["video2idx"][g["vid_name"]]
            ts = np.array(g["ts"], dtype=np.float32)
            inter = np.maximum(0, np.minimum(pr[:, 2], ts[1]) - np.maximum(pr[:, 1], ts[0]))
            union = np.maximum(pr[:, 2], ts[1]) - np.minimum(pr[:, 1], ts[0])
            iou = np.divide(inter, union, out=np.zeros_like(inter), where=union != 0) * match
            for thd in thds:
                c = iou >= thd
                if task == "SVMR":
                    c = c[match]
                for k in (1, 5, 10, 100):
                    hits[(thd, k)].append(match[:k].any() if task == "VR" else c[:k].any())
        res[task] = {f"{t}-r{k}": round(float(np.mean(v)) * 100, 2) for (t, k), v in hits.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2000)
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tvr_eval_probe needs a CUDA device")
    name, power = card()
    corpus, batches, video_ids, video2idx, gt, m, p, w = _setup(a.clips, a.queries)
    kw = dict(q2c_alpha=ALPHA, max_vcmr_video=K, min_pred_l=MIN_L, max_pred_l=MAX_L,
              max_before_nms=N, vfeat_interval=INTERVAL)
    n_in = min(N, MAX_AFTER_NMS)

    # NMS kernel time per batch of 80 (VCMR + SVMR lists of one ranked batch)
    out = evalpass.rank_modularized(corpus, m[:B], p[:B], w[0], w[1], q2c_alpha=ALPHA,
                                    max_video=K, min_pred_l=MIN_L, max_pred_l=MAX_L,
                                    max_before_nms=N, gt_vidx=torch.arange(B, device="cuda"))

    def nms_batch():
        for t, by_clip in (("VCMR", True), ("SVMR", False)):
            evalpass.nms_moments(*out[t], nms_thd=NMS_THD, n_in=n_in, n_out=n_in,
                                 interval=INTERVAL, by_clip=by_clip)
    for _ in range(5):
        nms_batch()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(a.iters):
        nms_batch()
    t1.record()
    torch.cuda.synchronize()
    nms_ms = t0.elapsed_time(t1) / a.iters

    # warm-up of both full paths on two batches
    evalpass.full_vcmr_eval(_Stub(), corpus, batches[:2], video_ids, video2idx,
                            [g for g in gt if g["desc_id"] < 2 * B], max_after_nms=MAX_AFTER_NMS,
                            nms_thd=NMS_THD, **kw)
    evalpass.full_vcmr_predictions(_Stub(), corpus, batches[:2], video_ids, video2idx, **kw)
    torch.cuda.synchronize()

    t = time.perf_counter()
    ours = evalpass.full_vcmr_eval(_Stub(), corpus, batches, video_ids, video2idx, gt,
                                   max_after_nms=MAX_AFTER_NMS, nms_thd=NMS_THD, **kw)
    ours_s = time.perf_counter() - t

    t = time.perf_counter()
    pred = evalpass.full_vcmr_predictions(_Stub(), corpus, batches, video_ids, video2idx, **kw)
    t_rank = time.perf_counter() - t
    sub = {k: v if k == "video2idx" else [dict(e, predictions=e["predictions"][:MAX_AFTER_NMS])
                                          for e in v] for k, v in pred.items()}
    host_metrics(sub, gt)
    nms = host_nms(sub, n_in)
    host_metrics(nms, gt)
    host_s = time.perf_counter() - t

    same_nms = all(ours["submission_nms"][k] == nms[k] for k in ("SVMR", "VCMR"))
    res = dict(card=name, power_limit_and_max_sm_clock=power, clips=a.clips, queries=a.queries,
               batch=B, K=K, N=N, max_after_nms=MAX_AFTER_NMS, nms_thd=NMS_THD,
               nms_kernel_ms_per_batch=round(nms_ms, 4),
               full_vcmr_eval_s=round(ours_s, 3),
               predictions_then_host_nms_metrics_s=round(host_s, 3),
               of_which_full_vcmr_predictions_s=round(t_rank, 3),
               nms_lists_identical=bool(same_nms),
               vcmr_metrics_nms=ours["metrics_nms"]["VCMR"])
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
