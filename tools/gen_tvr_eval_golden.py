"""Writes tests/golden/tvr_eval_tiny.npz: the reference's temporal NMS and TVR metrics on seeded
ranked moment lists.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_tvr_eval_golden.py

The inputs are ranked lists in the layout of `evalpass.rank_modularized` (score (Nq, N), moments
(Nq, N, 3) = clip row, start, end frame, descending score, padded with -1) and VR lists (score,
clip row). They are turned into submission records by `evalpass._submission` (the builder of
`full_vcmr_eval` and `full_*_predictions`) and fed to the reference's own utils/tvr_eval_utils.py
and utils/tvr_standalone_eval.py, imported from the checkout. Stored outputs (JSON strings):

* nms_vcmr / nms_svmr: post_processing_{vcmr,svmr}_nms of every row's first N_IN entries;
* flow: eval_vcmr.py:420-481 run as written on the rows with a non-empty list (get_submission_top_n
  truncating eval_res in place, eval_retrieval, both NMS, eval_retrieval again), with the lists
  before NMS, after NMS, the eval_submission the reference returns, and both metric dicts.

The rows include exact score ties across clips, spans at IoU exactly NMS_THD, a clip with more than
100 NMS survivors, single-entry groups, fully padded rows and rows shorter than N_IN; the ground
truth has both `ts` forms (one pair, DiDeMo-style pairs) and desc types v / t / vt.
"""
import copy
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200.evalpass import _submission  # noqa: E402

NQ, NV, LD, K_VR = 24, 40, 200, 20
MAX_BEFORE_NMS, MAX_AFTER_NMS, NMS_THD, INTERVAL = LD, 150, 0.5, 1.5
N_IN = min(MAX_BEFORE_NMS, MAX_AFTER_NMS)
SEED = 7


def ranked_row(rng, clips, n_valid, disjoint=False, tie_levels=None):
    """One descending list of n_valid moments over `clips`, padded to LD."""
    score = np.zeros(LD, dtype=np.float32)
    mom = np.full((LD, 3), -1, dtype=np.int32)
    if tie_levels:
        sc = rng.choice(np.arange(1, tie_levels + 1), n_valid).astype(np.float32) * 0.125
    else:
        sc = rng.random(n_valid).astype(np.float32)
    sc = -np.sort(-sc, kind="stable")
    if disjoint:                       # one-frame spans at distinct starts: IoU 0 pairwise
        s = rng.permutation(4 * n_valid)[:n_valid]
        e = s.copy()
    else:                              # short integer spans: many pairs at IoU exactly 0.5
        s = rng.integers(0, 40, n_valid)
        e = s + rng.integers(0, 8, n_valid)
    score[:n_valid] = sc
    mom[:n_valid] = np.stack([rng.choice(clips, n_valid), s, e], 1)
    return score, mom


def build_inputs(rng):
    vs, vm, ss, sm, gt_clip = [], [], [], [], []
    for q in range(NQ):
        g = int(rng.integers(0, NV))
        pool = rng.choice(NV, int(rng.integers(2, 9)), replace=False)
        if q % 3:
            pool[-1] = g                 # the GT clip among the ranked ones
        if q == 0:                     # ties across clips: A(5) B(4) B(3) A(3) ...
            vs_row = ranked_row(rng, pool[:2], LD, tie_levels=4)
        elif q == 1:                   # more than 100 survivors in one clip
            vs_row = ranked_row(rng, [g], LD, disjoint=True)
        elif q == 2:                   # single-entry groups: every moment a different clip
            vs_row = ranked_row(rng, np.arange(NV), NV)
            vs_row[1][:NV, 0] = rng.permutation(NV)
        elif q == 3:                   # fully padded
            vs_row = ranked_row(rng, pool, 0)
        elif q in (4, 5):              # shorter than N_IN
            vs_row = ranked_row(rng, pool, int(rng.integers(1, 60)))
        else:
            vs_row = ranked_row(rng, pool, LD, tie_levels=6 if q % 3 == 0 else None)
        if q == 6:                     # exact ties inside one clip and across clips
            vs_row[0][:] = np.where(vs_row[1][:, 0] >= 0, np.float32(0.5), np.float32(0))
        # SVMR: every moment on the query's clip
        if q == 1:
            sv = ranked_row(rng, [g], LD, disjoint=True)
        elif q == 4:
            sv = ranked_row(rng, [g], 1)
        elif q == 7:
            sv = ranked_row(rng, [g], 0)             # no band-valid span
        else:
            sv = ranked_row(rng, [g], LD, tie_levels=5 if q % 2 else None)
        vs.append(vs_row[0]), vm.append(vs_row[1]), ss.append(sv[0]), sm.append(sv[1])
        gt_clip.append(g)
    vr_idx = np.stack([rng.permutation(NV)[:K_VR] for _ in range(NQ)]).astype(np.int32)
    for q in range(0, NQ, 2):                        # the GT clip is often retrieved
        pos = int(rng.integers(0, 12))
        if gt_clip[q] not in vr_idx[q]:
            vr_idx[q, pos] = gt_clip[q]
    vr_score = -np.sort(-rng.random((NQ, K_VR)).astype(np.float32), axis=1)
    return (np.stack(vs), np.stack(vm), np.stack(ss), np.stack(sm), np.array(gt_clip),
            vr_score, vr_idx)


def ground_truth(rng, desc_ids, svmr_mom, gt_clip, video_ids):
    gt = []
    for i, (d, m, g) in enumerate(zip(desc_ids, svmr_mom, gt_clip)):
        valid = m[m[:, 0] >= 0]

        def span():
            if len(valid) and rng.random() < 0.8:      # a predicted span, sometimes widened
                s, e = valid[int(rng.integers(0, min(len(valid), 30)))][1:]
                e = e + int(rng.integers(0, 3))
            else:
                s = int(rng.integers(0, 40))
                e = s + int(rng.integers(0, 8))
            return [float(s * INTERVAL), float((e + 1) * INTERVAL)]

        ts = [span() for _ in range(4 + i % 2)] if i % 4 == 3 else span()
        gt.append(dict(desc_id=int(d), desc="", type=("v", "t", "vt")[i % 3],
                       vid_name=video_ids[int(g)], ts=ts))
    return gt


def main():
    ref = os.environ.get("HERO_REFERENCE")
    if not ref:
        raise SystemExit("set HERO_REFERENCE to a checkout of the reference")
    sys.path.insert(0, ref)
    from utils.tvr_eval_utils import (get_submission_top_n, post_processing_svmr_nms,
                                      post_processing_vcmr_nms)
    from utils.tvr_standalone_eval import eval_retrieval

    rng = np.random.default_rng(SEED)
    vs, vm, ss, sm, gt_clip, vr_score, vr_idx = build_inputs(rng)
    video_ids = [f"vid{r:03d}" for r in range(NV)]
    video2idx = {v: 7 * r + 3 for r, v in enumerate(video_ids)}
    desc_ids = [500 + q for q in range(NQ)]

    def submission(rows, n=LD, **lists):
        """The records of the queries `rows` for each task's (score, clip row / moment) lists,
        cut to their first n entries."""
        res = {t: (score[rows, :n], mom[rows, :n]) for t, (score, mom) in lists.items()}
        return _submission([desc_ids[q] for q in rows], [res], True, video_ids, video2idx,
                           INTERVAL, [(t, t) for t in lists])[0]

    # 1. NMS alone on every row (the reference's SVMR NMS cannot take an empty list)
    every = list(range(NQ))
    nms_vcmr = post_processing_vcmr_nms(
        submission(every, N_IN, VCMR=(vs, vm))["VCMR"],
        nms_thd=NMS_THD, max_before_nms=MAX_BEFORE_NMS, max_after_nms=MAX_AFTER_NMS)
    nms_svmr = []
    for e in submission(every, N_IN, SVMR=(ss, sm))["SVMR"]:
        if e["predictions"]:
            e = post_processing_svmr_nms([e], nms_thd=NMS_THD, max_before_nms=MAX_BEFORE_NMS,
                                         max_after_nms=MAX_AFTER_NMS)[0]
        nms_svmr.append(e)

    # 2. the evaluation flow of eval_vcmr.py:416-481 on the rows its eval_retrieval can take
    rows = [q for q in range(NQ) if vm[q, 0, 0] >= 0 and sm[q, 0, 0] >= 0]
    eval_res = submission(rows, SVMR=(ss, sm), VCMR=(vs, vm), VR=(vr_score, vr_idx))
    gt = ground_truth(rng, [desc_ids[q] for q in rows], sm[rows], gt_clip[rows], video_ids)
    # eval_retrieval on the untruncated lists (it reads their first 100), before any aliasing
    metrics_full = eval_retrieval(copy.deepcopy(eval_res), gt, iou_thds=(0.5, 0.7), verbose=False)
    eval_submission = get_submission_top_n(eval_res, top_n=MAX_AFTER_NMS)
    metrics = eval_retrieval(eval_submission, gt, iou_thds=(0.5, 0.7), match_number=True,
                             verbose=False, use_desc_type=True)
    submission = copy.deepcopy({k: v for k, v in eval_submission.items() if k != "video2idx"})
    after = dict(video2idx=eval_res["video2idx"])
    after["SVMR"] = post_processing_svmr_nms(eval_res["SVMR"], nms_thd=NMS_THD,
                                             max_before_nms=MAX_BEFORE_NMS,
                                             max_after_nms=MAX_AFTER_NMS)
    after["VCMR"] = post_processing_vcmr_nms(eval_res["VCMR"], nms_thd=NMS_THD,
                                             max_before_nms=MAX_BEFORE_NMS,
                                             max_after_nms=MAX_AFTER_NMS)
    metrics_nms = eval_retrieval(after, gt, iou_thds=(0.5, 0.7), match_number=True,
                                 verbose=False, use_desc_type=True)
    # other thresholds, without desc types
    metrics_no_type = eval_retrieval(submission | dict(video2idx=video2idx), gt,
                                     iou_thds=(0.3, 0.5), verbose=False, use_desc_type=False)
    flow = dict(rows=rows, ground_truth=gt, submission=submission,
                submission_nms={k: v for k, v in after.items() if k != "video2idx"},
                eval_submission={k: v for k, v in eval_submission.items() if k != "video2idx"},
                metrics=metrics, metrics_nms=metrics_nms, metrics_full=metrics_full,
                metrics_no_type=metrics_no_type)
    config = dict(max_before_nms=MAX_BEFORE_NMS, max_after_nms=MAX_AFTER_NMS, nms_thd=NMS_THD,
                  interval=INTERVAL, n_in=N_IN, seed=SEED, video_ids=video_ids,
                  video2idx=video2idx, desc_ids=desc_ids)
    assert len(nms_vcmr[1]["predictions"]) == 100     # the per-clip cap is reached
    assert len(nms_svmr[1]["predictions"]) == 100
    path = os.path.join(ROOT, "tests", "golden", "tvr_eval_tiny.npz")
    np.savez_compressed(path, vcmr_score=vs, vcmr_mom=vm, svmr_score=ss, svmr_mom=sm,
                        gt_clip=gt_clip, vr_score=vr_score, vr_idx=vr_idx,
                        nms_vcmr=json.dumps(nms_vcmr), nms_svmr=json.dumps(nms_svmr),
                        flow=json.dumps(flow), config=json.dumps(config))
    print(f"tvr_eval_tiny.npz: {NQ} queries, {len(rows)} in the flow, metrics "
          f"{json.dumps(metrics['VCMR'])}")


if __name__ == "__main__":
    main()
