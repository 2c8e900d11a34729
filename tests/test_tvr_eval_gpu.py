"""Temporal NMS on the GPU (hero_b200/csrc/nms.cu + evalpass): the kernel against the reference's
NMS outputs (tests/golden/tvr_eval_tiny.npz) and against its restatement (tests/fake_nms_ops.py)
on large random lists with ties, both modes and several thresholds, nms_moments without host
synchronisation, and full_vcmr_eval end to end from embed_video_corpus.

The kernel's shared memory is static (about 32 KB for 1024 entries, under the 48 KB default), so
there is no dynamic shared-memory limit whose first launch could differ."""
import json

import numpy as np
import pytest
import torch

from hero_b200 import evalpass, ops, synth
from tests import fake_nms_ops as ref
from tests import golden_util as gu
from tests.test_tvr_eval_cpu import (_fixture, _flow_batches, _records, _same_metrics,
                                     check_eval, expected_eval)

pytestmark = pytest.mark.gpu
F32, I32 = torch.float32, torch.int32


def _nms(score, mom, n_in, thd, interval, by_clip, n_out):
    s = torch.full((score.shape[0], n_out), float("nan"), dtype=F32, device="cuda")
    m = torch.full((score.shape[0], n_out, 3), -7, dtype=I32, device="cuda")
    ops.temporal_nms(score, mom, n_in, thd, interval, by_clip, n_out, s, m)
    return s.cpu().numpy(), m.cpu().numpy()


@pytest.mark.parametrize("task", ["VCMR", "SVMR"])
def test_kernel_matches_reference_nms(task):
    fx, cfg, _ = _fixture()
    key = task.lower()
    want = json.loads(str(fx[f"nms_{key}"]))
    s, m = _nms(torch.from_numpy(fx[f"{key}_score"]).cuda(), torch.from_numpy(fx[f"{key}_mom"]).cuda(),
                cfg["n_in"], cfg["nms_thd"], cfg["interval"], task == "VCMR", cfg["max_after_nms"])
    for q, w in enumerate(want):
        got = _records(s[q], m[q], cfg, task == "SVMR")
        assert got == w["predictions"], q
        assert (s[q, len(got):] == 0).all() and (m[q, len(got):] == -1).all()


def _random_lists(nq, ld, n_pool, seed):
    """Descending lists with exact ties, clips from a pool of up to n_pool, short integer spans
    (many pairs at IoU exactly 1/2, 1/3, 2/3 ...) and padded tails."""
    rng = np.random.default_rng(seed)
    score = np.round(rng.random((nq, ld)) * 40).astype(np.float32) / 40
    score = -np.sort(-score, axis=1)
    clips = rng.integers(0, 1000, (nq, n_pool))[np.arange(nq)[:, None],
                                                 rng.integers(0, n_pool, (nq, ld))]
    s = rng.integers(0, 100, (nq, ld))
    e = s + rng.integers(0, 12, (nq, ld))
    mom = np.stack([clips, s, e], -1).astype(np.int32)
    n_valid = np.where(rng.random(nq) < 0.1, rng.integers(0, ld + 1, nq), ld)
    pad = np.arange(ld)[None, :] >= n_valid[:, None]
    score[pad] = 0
    mom[pad] = -1
    return score, mom


@pytest.mark.parametrize("by_clip", [True, False])
@pytest.mark.parametrize("n_in", [100, 200, 1024])
def test_kernel_matches_restatement_on_large_inputs(by_clip, n_in):
    nq, ld = 1000, min(1024, n_in + 8)
    score, mom = _random_lists(nq, ld, 12 if by_clip else 1, seed=n_in + by_clip)
    ds, dm = torch.from_numpy(score).cuda(), torch.from_numpy(mom).cuda()
    for thd in (0.3, 0.5, 0.7):
        n_out = min(n_in, 150)
        s, m = _nms(ds, dm, n_in, thd, 1.5, by_clip, n_out)
        rs, rm = ref.nms_ref(score, mom, n_in, thd, 1.5, by_clip, n_out)
        assert np.array_equal(m, rm), thd
        assert np.array_equal(s, rs), thd


def test_kernel_group_cap_and_argument_checks():
    # 300 disjoint one-frame spans of one clip: 100 kept per group in both modes
    ld = 300
    score = torch.linspace(1, 0, ld).view(1, ld).cuda()
    mom = torch.stack([torch.full((ld,), 3), torch.arange(ld), torch.arange(ld)], -1)
    mom = mom.to(I32).view(1, ld, 3).cuda()
    for by_clip in (True, False):
        s, m = _nms(score, mom, ld, 0.5, 1.0, by_clip, 200)
        assert (m[0, :100, 1] == np.arange(100)).all() and (m[0, 100:] == -1).all()
    out_s, out_m = torch.empty(1, 10, device="cuda"), torch.empty(1, 10, 3, dtype=I32, device="cuda")
    for args in ((1025, 10), (10, 0), (10, 1025)):
        with pytest.raises(Exception, match="temporal_nms"):
            n_in, n_out = args
            ops.temporal_nms(score, mom, n_in, 0.5, 1.0, True, n_out, out_s, out_m)


def test_nms_moments_does_not_synchronise():
    score, mom = _random_lists(80, 200, 8, seed=3)
    ds, dm = torch.from_numpy(score).cuda(), torch.from_numpy(mom).cuda()
    evalpass.nms_moments(ds, dm, nms_thd=0.5, n_in=100, n_out=100, interval=1.5, by_clip=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        s, m = evalpass.nms_moments(ds, dm, nms_thd=0.5, n_in=100, n_out=100, interval=1.5,
                                    by_clip=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    rs, rm = ref.nms_ref(score, mom, 100, 0.5, 1.5, True, 100)
    assert np.array_equal(m.cpu().numpy(), rm) and np.array_equal(s.cpu().numpy(), rs)


def test_full_vcmr_eval_flow_on_the_kernel(monkeypatch):
    """The reference flow of the fixture with the real kernel (ranking replaced by the lists)."""
    fx, cfg, flow = _fixture()
    batches, rank_queries = _flow_batches(fx, cfg, flow["rows"])

    def rank_on_gpu(*a, **kw):
        return {k: tuple(t.cuda() for t in v) for k, v in rank_queries(*a, **kw).items()}
    monkeypatch.setattr(evalpass, "rank_queries", rank_on_gpu)
    corpus = evalpass.VideoCorpus(torch.randn(len(cfg["video_ids"]), 4, 8).cuda(),
                                  torch.ones(len(cfg["video_ids"]), 4).cuda())

    class Stub(torch.nn.Module):
        lw_neg_ctx = lw_neg_q = 8
    res = evalpass.full_vcmr_eval(Stub(), corpus, batches, cfg["video_ids"], cfg["video2idx"],
                                  flow["ground_truth"], max_before_nms=cfg["max_before_nms"],
                                  max_after_nms=cfg["max_after_nms"], nms_thd=cfg["nms_thd"],
                                  vfeat_interval=cfg["interval"])
    for k in ("SVMR", "VCMR"):
        assert res["submission_nms"][k] == flow["submission_nms"][k], k
    _same_metrics(res["metrics"], flow["metrics"])
    _same_metrics(res["metrics_nms"], flow["metrics_nms"])


def test_full_vcmr_eval_end_to_end_from_embed_video_corpus(tmp_path):
    from tests.test_heads_cpu import _vcmr_model
    model, _, vx = _vcmr_model(tmp_path)
    model = model.cuda().eval()
    d = gu.dims_of(gu.load("hier_tiny.npz"))
    vbs = [synth.syn_tvr_ragged(batch_size=4, seed=70 + i, vfeat_dim=d["vfeat_dim"],
                                vocab=d["vocab"] - 7, t_range=t, s_range=(2, 4), l_range=(3, 8),
                                q_range=(3, 7))[0] for i, t in enumerate([(2, 9), (12, 20)])]
    emb, masks = evalpass.embed_video_corpus(model, vbs, n_videos=8, max_clip_len=20)
    corpus = evalpass.VideoCorpus(emb, masks)
    nq = vx["query_input_ids"].shape[0]
    video_ids = [f"v{i}" for i in range(8)]
    video2idx = {v: 10 + i for i, v in enumerate(video_ids)}
    gt_clip = [i % 8 for i in range(nq)]
    batch = dict(qids=list(range(nq)), vids=[video_ids[g] for g in gt_clip],
                 targets=torch.zeros(nq, 2, dtype=torch.long),
                 query_input_ids=torch.from_numpy(vx["query_input_ids"]),
                 query_pos_ids=torch.from_numpy(vx["query_pos_ids"]),
                 query_attn_masks=torch.from_numpy(vx["query_attn_masks"]))
    gt = [dict(desc_id=q, desc="", type=("v", "t", "vt")[q % 3], vid_name=video_ids[gt_clip[q]],
               ts=[float(q % 4), float(q % 4 + 3)] if q % 4 != 3 else
               [[0.0, 2.0], [1.0, 3.0], [0.0, 4.0], [2.0, 5.0]]) for q in range(nq)]
    kw = dict(q2c_alpha=20.0, max_vcmr_video=5, min_pred_l=1, max_pred_l=6, max_before_nms=40,
              vfeat_interval=1.0)
    res = evalpass.full_vcmr_eval(model, corpus, [batch], video_ids, video2idx, gt,
                                  max_after_nms=30, nms_thd=0.5, **kw)
    pred = evalpass.full_vcmr_predictions(model, corpus, [batch], video_ids, video2idx, **kw)
    check_eval(res, expected_eval(pred, gt, video_ids, video2idx, 30, 0.5, 1.0))
