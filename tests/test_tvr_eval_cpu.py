"""Temporal NMS and TVR metrics (evalpass.nms_moments / eval_retrieval / full_vcmr_eval) on the CPU,
with the NMS kernel replaced by its plain restatement (tests/fake_nms_ops.py). The expected lists
and metric dicts are the reference's own (tests/golden/tvr_eval_tiny.npz,
tools/gen_tvr_eval_golden.py) and are compared with ==: the same entries in the same order, the
same floats, the same OrderedDicts. The kernel itself is covered by tests/test_tvr_eval_gpu.py."""
import copy
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch import nn

from hero_b200 import evalpass
from tests import fake_nms_ops, fake_rank_ops
from tests import golden_util as gu
from tests.test_retrieval_cpu import _batches as _rank_batches
from tests.test_retrieval_cpu import _corpus, _golden, _StubQueryModel


def _fixture():
    fx = gu.load("tvr_eval_tiny.npz")
    return fx, json.loads(str(fx["config"])), json.loads(str(fx["flow"]))


def _same_metrics(got, want):
    assert json.dumps(got) == json.dumps(want)          # keys, order and float reprs
    assert got == want
    for task in got.values():
        for v in task.values():
            assert isinstance(v, (float, str))


def _records(score, mom, cfg, svmr):
    return evalpass._moment_records(score, mom, cfg["video_ids"], cfg["video2idx"],
                                    cfg["interval"], svmr)


@pytest.mark.parametrize("task", ["VCMR", "SVMR"])
def test_nms_moments_match_reference_nms(monkeypatch, task):
    fake_nms_ops.install(monkeypatch)
    fx, cfg, _ = _fixture()
    key = task.lower()
    want = json.loads(str(fx[f"nms_{key}"]))
    score, mom = torch.from_numpy(fx[f"{key}_score"]), torch.from_numpy(fx[f"{key}_mom"])
    s, m = evalpass.nms_moments(score, mom, nms_thd=cfg["nms_thd"], n_in=cfg["n_in"],
                                n_out=cfg["max_after_nms"], interval=cfg["interval"],
                                by_clip=task == "VCMR")
    assert s.shape == (len(score), cfg["max_after_nms"])
    for q, w in enumerate(want):
        got = _records(s[q].numpy(), m[q].numpy(), cfg, task == "SVMR")
        assert got == w["predictions"], q
        n = len(got)
        assert (s[q, n:] == 0).all() and (m[q, n:] == -1).all()


class _StubModel(nn.Module):
    lw_neg_ctx = lw_neg_q = 8


def _flow_batches(fx, cfg, rows, split=(9, 13)):
    """Query batches whose `query_input_ids[:, 0]` is the fixture row, and a rank_queries that
    returns that row's ranked lists."""
    vid = cfg["video_ids"]
    out, a = [], 0
    for n in split:
        r = rows[a:a + n]
        out.append(dict(qids=[cfg["desc_ids"][q] for q in r],
                        vids=[vid[int(fx["gt_clip"][q])] for q in r],
                        targets=torch.zeros(len(r), 2, dtype=torch.long),
                        query_input_ids=torch.tensor(r)[:, None],
                        query_pos_ids=torch.zeros(1, 1, dtype=torch.long),
                        query_attn_masks=torch.ones(len(r), 1, dtype=torch.long)))
        a += n
    assert a == len(rows)

    def rank_queries(model, corpus, qb, *, tasks, gt_vidx=None, **kw):
        r = qb["query_input_ids"][:, 0].long().cpu().numpy()
        t = {"VR": ("vr_score", "vr_idx"), "VCMR": ("vcmr_score", "vcmr_mom"),
             "SVMR": ("svmr_score", "svmr_mom")}
        return {k: tuple(torch.from_numpy(fx[n][r]) for n in t[k]) for k in tasks}
    return out, rank_queries


def _flow_eval(monkeypatch, fx, cfg, flow, **kw):
    fake_rank_ops.install(monkeypatch)
    fake_nms_ops.install(monkeypatch)
    batches, rank_queries = _flow_batches(fx, cfg, flow["rows"])
    monkeypatch.setattr(evalpass, "rank_queries", rank_queries)
    args = dict(max_before_nms=cfg["max_before_nms"], max_after_nms=cfg["max_after_nms"],
                nms_thd=cfg["nms_thd"], vfeat_interval=cfg["interval"])
    args.update(kw)
    return evalpass.full_vcmr_eval(_StubModel(), SimpleNamespace(device="cpu"), batches,
                                   cfg["video_ids"], cfg["video2idx"], flow["ground_truth"], **args)


def test_full_vcmr_eval_reproduces_the_reference_flow(monkeypatch):
    fx, cfg, flow = _fixture()
    res = _flow_eval(monkeypatch, fx, cfg, flow)
    assert list(res) == ["submission", "metrics", "submission_nms", "metrics_nms"]
    sub, sub_nms = res["submission"], res["submission_nms"]
    assert list(sub) == ["SVMR", "VCMR", "VR", "video2idx"]
    assert list(sub_nms) == ["SVMR", "VCMR", "video2idx"]
    assert sub["video2idx"] is cfg["video2idx"] or sub["video2idx"] == cfg["video2idx"]
    for k in ("SVMR", "VCMR", "VR"):
        assert sub[k] == flow["submission"][k], k
    for k in ("SVMR", "VCMR"):
        assert sub_nms[k] == flow["submission_nms"][k], k
    # what the reference returns: its eval_res lists, NMS'd in place
    assert dict(SVMR=sub_nms["SVMR"], VCMR=sub_nms["VCMR"], VR=sub["VR"]) == \
        flow["eval_submission"]
    _same_metrics(res["metrics"], flow["metrics"])
    _same_metrics(res["metrics_nms"], flow["metrics_nms"])


def test_full_vcmr_eval_without_nms_or_ground_truth(monkeypatch):
    fx, cfg, flow = _fixture()
    res = _flow_eval(monkeypatch, fx, cfg, flow, nms_thd=-1)
    assert list(res) == ["submission", "metrics"]
    _same_metrics(res["metrics"], flow["metrics"])
    res = _flow_eval(monkeypatch, fx, cfg, dict(flow, ground_truth=None))
    assert list(res) == ["submission", "submission_nms"]
    assert res["submission_nms"]["VCMR"] == flow["submission_nms"]["VCMR"]


def test_eval_retrieval_matches_reference(monkeypatch):
    fx, cfg, flow = _fixture()
    v2i, gt = cfg["video2idx"], flow["ground_truth"]
    sub = dict(flow["submission"], video2idx=v2i)
    _same_metrics(evalpass.eval_retrieval(sub, gt), flow["metrics"])
    _same_metrics(evalpass.eval_retrieval(dict(flow["submission_nms"], video2idx=v2i), gt),
                  flow["metrics_nms"])
    _same_metrics(evalpass.eval_retrieval(sub, gt, iou_thds=(0.3, 0.5), use_desc_type=False),
                  flow["metrics_no_type"])
    # the untruncated lists (200 moments): only the first 100 count
    rows = flow["rows"]
    full = dict(video2idx=v2i)
    for task, svmr in (("SVMR", True), ("VCMR", False)):
        key = task.lower()
        full[task] = [dict(desc_id=cfg["desc_ids"][q], desc="", predictions=_records(
            fx[f"{key}_score"][q], fx[f"{key}_mom"][q], cfg, svmr)) for q in rows]
    full["VR"] = sub["VR"]
    _same_metrics(evalpass.eval_retrieval(full, gt), flow["metrics_full"])
    # prediction order and query order of the submission do not matter beyond the top 100
    shuffled = dict(sub, VCMR=list(reversed(sub["VCMR"])))
    _same_metrics(evalpass.eval_retrieval(shuffled, list(reversed(gt))), flow["metrics"])


def test_eval_retrieval_errors():
    _, cfg, flow = _fixture()
    sub = dict(flow["submission"], video2idx=cfg["video2idx"])
    gt = copy.deepcopy(flow["ground_truth"])
    with pytest.raises(ValueError, match="must match"):
        evalpass.eval_retrieval(sub, gt[1:])
    evalpass.eval_retrieval(sub, gt[1:], match_number=False)
    for n_pairs in (2, 3):
        bad = copy.deepcopy(gt)
        bad[0]["ts"] = [[0.0, 1.5]] * n_pairs
        with pytest.raises(ValueError, match="ts"):
            evalpass.eval_retrieval(sub, bad)
    bad = copy.deepcopy(gt)
    bad[0]["type"] = "x"
    with pytest.raises(ValueError, match="desc types"):
        evalpass.eval_retrieval(sub, bad)
    evalpass.eval_retrieval(sub, bad, use_desc_type=False)


def test_nms_moments_errors_and_empty_rows(monkeypatch):
    fake_nms_ops.install(monkeypatch)
    score = torch.zeros(2, 10)
    mom = torch.full((2, 10, 3), -1, dtype=torch.int32)
    mom[0, :3] = torch.tensor([[4, 0, 2], [4, 1, 2], [4, 5, 6]], dtype=torch.int32)
    score[0, :3] = torch.tensor([0.9, 0.8, 0.7])
    kw = dict(nms_thd=0.5, interval=1.5, by_clip=False)
    with pytest.raises(ValueError, match="n_in"):
        evalpass.nms_moments(score, mom, n_in=11, n_out=5, **kw)
    with pytest.raises(ValueError, match="n_out"):
        evalpass.nms_moments(score, mom, n_in=10, n_out=0, **kw)
    s, m = evalpass.nms_moments(score, mom, n_in=10, n_out=5, **kw)
    # [0, 4.5] vs [1.5, 4.5]: IoU 2/3 > 0.5, dropped; an empty row stays empty (no IndexError)
    assert m[0, :, 1].tolist() == [0, 5, -1, -1, -1] and torch.equal(s[0, :2], score[0, [0, 2]])
    assert (m[1] == -1).all() and (s[1] == 0).all()
    s, m = evalpass.nms_moments(score, mom, n_in=1, n_out=5, **kw)
    assert m[0, :, 1].tolist() == [0, -1, -1, -1, -1]


def test_vcmr_merge_ties_follow_first_appearance():
    """A(5) B(4) B(3) A(3) -> A B A B: equal scores go to the clip seen first."""
    score = np.array([[5, 4, 3, 3]], dtype=np.float32)
    mom = np.array([[[0, 0, 1], [1, 0, 1], [1, 10, 11], [0, 10, 11]]], dtype=np.int32)
    s, m = fake_nms_ops.nms_ref(score, mom, 4, 0.5, 1.5, True, 4)
    assert m[0, :, 0].tolist() == [0, 1, 0, 1] and s[0].tolist() == [5, 4, 3, 3]


# ------------------------------------------------------------------ end to end
def _rank_ground_truth(fx, video_ids, n_pairs_every=4):
    """Ground truth for the queries of vcmr_rank_tiny.npz: the GT clip, desc types v / t / vt,
    spans in seconds, DiDeMo-style pairs for every fourth query."""
    gt = []
    for q in range(len(fx["m"])):
        s = 1.5 * (q % 5)
        span = [s, s + 3.0]
        ts = [span, [s, s + 1.5], [0.0, 6.0], span] if q % n_pairs_every == 3 else span
        gt.append(dict(desc_id=100 + q, desc="", type=("v", "t", "vt")[q % 3],
                       vid_name=video_ids[int(fx["gt_vidx"][q])], ts=ts))
    return gt


def _truncated(eval_res, n):
    return {k: v if k == "video2idx" else [dict(e, predictions=e["predictions"][:n]) for e in v]
            for k, v in eval_res.items()}


def expected_eval(pred, gt, video_ids, video2idx, n_after, thd, interval):
    """full_vcmr_eval restated from full_vcmr_predictions' eval_res: get_submission_top_n, the NMS
    restatement on each list, eval_retrieval before and after."""
    want = _truncated(pred, n_after)
    out = dict(submission=want, metrics=evalpass.eval_retrieval(want, gt))
    row = {video2idx[v]: i for i, v in enumerate(video_ids)}
    nms = dict(video2idx=video2idx)
    for task, by_clip in (("SVMR", False), ("VCMR", True)):
        lists = []
        for e in want[task]:
            p = e["predictions"]
            mom = np.array([[row[r[0]], round(r[1] / interval), round(r[2] / interval) - 1]
                            for r in p], np.int32).reshape(1, -1, 3)
            sc = np.array([[r[3] for r in p]], np.float32)
            s, m = fake_nms_ops.nms_ref(sc, mom, len(p), thd, interval, by_clip, max(1, len(p)))
            lists.append(dict(e, predictions=evalpass._moment_records(
                s[0], m[0], video_ids, video2idx, interval, not by_clip)))
        nms[task] = lists
    out.update(submission_nms=nms, metrics_nms=evalpass.eval_retrieval(nms, gt))
    return out


def check_eval(res, want):
    assert list(res) == ["submission", "metrics", "submission_nms", "metrics_nms"]
    for k in ("SVMR", "VCMR", "VR"):
        assert res["submission"][k] == want["submission"][k], k
    for k in ("SVMR", "VCMR"):
        assert res["submission_nms"][k] == want["submission_nms"][k], k
    _same_metrics(res["metrics"], want["metrics"])
    _same_metrics(res["metrics_nms"], want["metrics_nms"])


def test_full_vcmr_eval_end_to_end(monkeypatch):
    """full_vcmr_eval == full_vcmr_predictions, truncated, then the NMS restatement and
    eval_retrieval, on the ranking golden with a stub query model."""
    fake_rank_ops.install(monkeypatch)
    fake_nms_ops.install(monkeypatch)
    fx, cfg = _golden()
    batches, video_ids, video2idx = _rank_batches(fx)
    gt = _rank_ground_truth(fx, video_ids)
    kw = dict(q2c_alpha=cfg["q2c_alpha"], max_vcmr_video=cfg["K"], min_pred_l=cfg["min_pred_l"],
              max_pred_l=cfg["max_pred_l"], max_before_nms=cfg["N"], vfeat_interval=1.5)
    res = evalpass.full_vcmr_eval(_StubQueryModel(fx), _corpus(fx), batches, video_ids,
                                  video2idx, gt, max_after_nms=20, nms_thd=0.5, **kw)
    pred = evalpass.full_vcmr_predictions(_StubQueryModel(fx), _corpus(fx), batches, video_ids,
                                          video2idx, **kw)
    check_eval(res, expected_eval(pred, gt, video_ids, video2idx, 20, 0.5, 1.5))
