"""Full-corpus retrieval ranking (evalpass.rank_queries / full_vcmr_predictions /
full_vr_predictions) and HeroForVr, on the CPU with hero_b200.ops routed through the torch
restatements (tests/fake_ops.py, tests/fake_rank_ops.py). The expected lists come from the
reference's HeroForVcmr head (tests/golden/vcmr_rank_tiny.npz, tools/gen_rank_golden.py); the
kernels themselves are covered by tests/test_retrieval_gpu.py."""
import json

import numpy as np
import pytest
import torch
from torch import nn

from hero_b200 import evalpass
from tests import fake_rank_ops
from tests import golden_util as gu

INTERVAL = 1.5


def _golden():
    fx = gu.load("vcmr_rank_tiny.npz")
    return fx, json.loads(str(fx["config"]))


def _corpus(fx):
    return evalpass.VideoCorpus(torch.from_numpy(fx["frames"]), torch.from_numpy(fx["c_attn_masks"]))


def _rank_kw(cfg, **kw):
    d = dict(q2c_alpha=cfg["q2c_alpha"], max_video=cfg["K"], min_pred_l=cfg["min_pred_l"],
             max_pred_l=cfg["max_pred_l"], max_before_nms=cfg["N"])
    d.update(kw)
    return d


def _same_ranking(got_s, got_keys, ref_s, ref_keys):
    """Scores equal at every sorted rank within 1e-4 * max|ref|; the same set of entries."""
    tol = 1e-4 * float(np.abs(ref_s).max())
    assert len(got_s) == len(ref_s)
    assert np.abs(np.asarray(got_s, np.float64) - np.asarray(ref_s, np.float64)).max() <= tol
    assert sorted(map(tuple, np.asarray(got_keys).reshape(len(got_keys), -1).tolist())) == \
        sorted(map(tuple, np.asarray(ref_keys).reshape(len(ref_keys), -1).tolist()))


def test_rank_modularized_matches_reference(monkeypatch):
    fake_rank_ops.install(monkeypatch)
    fx, cfg = _golden()
    corpus = _corpus(fx)
    out = evalpass.rank_modularized(
        corpus, torch.from_numpy(fx["m"]), torch.from_numpy(fx["p"]), torch.from_numpy(fx["w_st"]),
        torch.from_numpy(fx["w_ed"]), gt_vidx=torch.from_numpy(fx["gt_vidx"]), **_rank_kw(cfg))
    vs, vi = (t.numpy() for t in out["VR"])
    ms, mm = (t.numpy() for t in out["VCMR"])
    ss, sm = (t.numpy() for t in out["SVMR"])
    for q in range(len(fx["m"])):
        _same_ranking(vs[q], vi[q], fx["vr_scores"][q], fx["vr_idx"][q])
        _same_ranking(ms[q], mm[q], fx["vcmr_scores"][q], fx["vcmr_moments"][q])
        tri = fx["svmr_triples"][q]
        ref_keys = np.stack([np.full(len(tri), fx["gt_vidx"][q]), tri[:, 0], tri[:, 1]], 1)
        _same_ranking(ss[q], sm[q], tri[:, 2], ref_keys.astype(np.int64))
    raw = evalpass.rank_modularized(corpus, torch.from_numpy(fx["m"]), None, None, None,
                                    tasks=("VR",), max_video=cfg["K_VR"])
    for q in range(len(fx["m"])):
        _same_ranking(raw["VR"][0][q].numpy(), raw["VR"][1][q].numpy(), fx["vr_raw_scores"][q],
                      fx["vr_raw_idx"][q])


class _StubQueryModel(nn.Module):
    """Stands in for the text encoder + query pooling: query_input_ids[:, 0] picks a stored
    modularized query, so the ranking half runs on the golden's queries."""

    def __init__(self, fx, lw=8):
        super().__init__()
        m = torch.from_numpy(fx["m"])
        self.register_buffer("m", m)
        vx = gu.load("vsm_tiny.npz")
        self.video_query_linear = nn.Linear(m.shape[1], m.shape[1])
        self.video_query_linear.weight.data.copy_(torch.from_numpy(vx["head.video_query_linear.weight"]))
        self.video_query_linear.bias.data.copy_(torch.from_numpy(vx["head.video_query_linear.bias"]))
        conv = dict(in_channels=1, out_channels=1, kernel_size=5, padding=2, bias=False)
        self.video_st_predictor, self.video_ed_predictor = nn.Conv1d(**conv), nn.Conv1d(**conv)
        self.video_st_predictor.weight.data.copy_(torch.from_numpy(fx["w_st"]).view(1, 1, 5))
        self.video_ed_predictor.weight.data.copy_(torch.from_numpy(fx["w_ed"]).view(1, 1, 5))
        self.lw_neg_ctx = self.lw_neg_q = lw

    def q_feat_attn(self, feats, mask):
        return feats[:, 0]

    def encode_txt_inputs(self, input_ids, pos_ids, attn_masks, attn_layer=None,
                          normalized=False, plan=None):
        assert attn_layer == self.q_feat_attn and not normalized and plan is not None
        return attn_layer(self.m[input_ids[:, 0]].unsqueeze(1), attn_masks)


def _batches(fx, split=(6, 4), targets_ok=True):
    video_ids = [f"clip{i:02d}" for i in range(len(fx["frames"]))]
    out, q0 = [], 0
    for n in split:
        ids = torch.arange(q0, q0 + n)[:, None]
        out.append(dict(qids=[100 + q for q in range(q0, q0 + n)],
                        vids=[video_ids[int(fx["gt_vidx"][q])] for q in range(q0, q0 + n)],
                        targets=torch.zeros(n, 2, dtype=torch.long) - (0 if targets_ok else 1),
                        query_input_ids=ids, query_pos_ids=torch.zeros(1, 1, dtype=torch.long),
                        query_attn_masks=torch.ones(n, 1, dtype=torch.long)))
        q0 += n
    video2idx = {v: 1000 + 3 * i for i, v in enumerate(video_ids)}
    return out, video_ids, video2idx


def _expected_eval_res(fx, cfg, video_ids, video2idx):
    """eval_res as eval_vcmr.py:325-418 builds it from the golden's lists."""
    L = fx["frames"].shape[1]
    svmr, vcmr, vr = [], [], []
    for q in range(len(fx["m"])):
        vid = video2idx[video_ids[int(fx["gt_vidx"][q])]]
        tri = fx["svmr_triples"][q].copy()
        tri[:, 1] += 1
        tri[:, :2] *= INTERVAL
        svmr.append(dict(desc_id=100 + q, desc="", predictions=[[vid] + r for r in tri.tolist()]))
        vr.append(dict(desc_id=100 + q, desc="", predictions=[
            [video2idx[video_ids[int(i)]], 0, 0, float(s)]
            for s, i in zip(fx["vr_scores"][q][:100], fx["vr_idx"][q][:100])]))
        mom = fx["vcmr_moments"][q]
        st = mom[:, 1].astype(np.float32) * INTERVAL
        ed = mom[:, 2].astype(np.float32) * INTERVAL + INTERVAL
        vcmr.append(dict(desc_id=100 + q, desc="", predictions=[
            [video2idx[video_ids[int(mom[i, 0])]], float(st[i]), float(ed[i]),
             float(fx["vcmr_scores"][q][i])] for i in range(len(mom))]))
    assert L == fx["c_attn_masks"].shape[1]
    return dict(SVMR=svmr, VCMR=vcmr, VR=vr)


def _same_records(got, ref):
    assert [r["desc_id"] for r in got] == [r["desc_id"] for r in ref]
    for g, r in zip(got, ref):
        assert g["desc"] == "" and type(g["desc_id"]) is type(r["desc_id"])
        gp, rp = g["predictions"], r["predictions"]
        _same_ranking([p[3] for p in gp], [p[:3] for p in gp], [p[3] for p in rp],
                      [p[:3] for p in rp])
        for p in gp:       # [video_idx (int), st (float), ed (float), score (float)]
            assert type(p[0]) is int and all(type(x) in (float, int) for x in p[1:])


def test_full_vcmr_predictions_match_reference_eval_res(monkeypatch):
    fake_rank_ops.install(monkeypatch)
    fx, cfg = _golden()
    batches, video_ids, video2idx = _batches(fx)
    res = evalpass.full_vcmr_predictions(
        _StubQueryModel(fx), _corpus(fx), batches, video_ids, video2idx,
        q2c_alpha=cfg["q2c_alpha"], max_vcmr_video=cfg["K"], min_pred_l=cfg["min_pred_l"],
        max_pred_l=cfg["max_pred_l"], max_before_nms=cfg["N"], vfeat_interval=INTERVAL)
    ref = _expected_eval_res(fx, cfg, video_ids, video2idx)
    assert list(res) == ["SVMR", "VCMR", "VR", "video2idx"]
    assert res["video2idx"] is video2idx
    for k in ("SVMR", "VCMR", "VR"):
        _same_records(res[k], ref[k])
    # the seconds are exact: start = s * interval, end = (e + 1) * interval
    for got, r in zip(res["SVMR"], ref["SVMR"]):
        assert sorted(p[:3] for p in got["predictions"]) == sorted(p[:3] for p in r["predictions"])
    for got, r in zip(res["VCMR"], ref["VCMR"]):
        assert sorted(p[:3] for p in got["predictions"]) == sorted(p[:3] for p in r["predictions"])


def test_full_vcmr_predictions_drops_empty_tasks(monkeypatch):
    fake_rank_ops.install(monkeypatch)
    fx, cfg = _golden()
    kw = dict(q2c_alpha=cfg["q2c_alpha"], max_vcmr_video=cfg["K"], min_pred_l=cfg["min_pred_l"],
              max_pred_l=cfg["max_pred_l"], max_before_nms=cfg["N"], vfeat_interval=INTERVAL)
    batches, video_ids, video2idx = _batches(fx, targets_ok=False)       # no ground truth
    res = evalpass.full_vcmr_predictions(_StubQueryModel(fx), _corpus(fx), batches, video_ids,
                                         video2idx, **kw)
    assert list(res) == ["VCMR", "VR", "video2idx"]
    batches, video_ids, video2idx = _batches(fx)
    res = evalpass.full_vcmr_predictions(_StubQueryModel(fx, lw=0), _corpus(fx), batches,
                                         video_ids, video2idx, **kw)      # no video-level scores
    assert list(res) == ["SVMR", "video2idx"]
    res = evalpass.full_vcmr_predictions(_StubQueryModel(fx), _corpus(fx), batches, video_ids,
                                         video2idx, tasks=("VCMR",), **kw)   # VCMR needs VR
    assert list(res) == ["video2idx"]


def test_full_vr_predictions_match_reference(monkeypatch):
    fake_rank_ops.install(monkeypatch)
    fx, cfg = _golden()
    batches, video_ids, video2idx = _batches(fx, split=(3, 3, 4))
    res = evalpass.full_vr_predictions(_StubQueryModel(fx), _corpus(fx), batches, video_ids,
                                       video2idx, max_vr_video=cfg["K_VR"])
    assert list(res) == ["VR", "video2idx"]
    ref = [dict(desc_id=100 + q, desc="", predictions=[
        [video2idx[video_ids[int(i)]], 0, 0, float(s)]
        for s, i in zip(fx["vr_raw_scores"][q], fx["vr_raw_idx"][q])]) for q in range(len(fx["m"]))]
    _same_records(res["VR"], ref)


def test_rank_errors(monkeypatch):
    fake_rank_ops.install(monkeypatch)
    fx, cfg = _golden()
    corpus = _corpus(fx)
    m, p = torch.from_numpy(fx["m"]), torch.from_numpy(fx["p"])
    w = torch.from_numpy(fx["w_st"])
    gt = torch.from_numpy(fx["gt_vidx"])

    def call(**kw):
        args = dict(_rank_kw(cfg), gt_vidx=gt)
        args.update(kw)
        return evalpass.rank_modularized(corpus, m, p, w, w, **args)

    nv = fx["frames"].shape[0]
    with pytest.raises(ValueError, match="max_video"):
        call(max_video=nv + 1)                      # torch.topk would fail too
    with pytest.raises(ValueError, match="max_before_nms"):
        call(max_before_nms=1025)
    with pytest.raises(ValueError, match="gt_vidx"):
        call(gt_vidx=None)
    with pytest.raises(ValueError, match="gt_vidx"):
        call(gt_vidx=[nv] * len(fx["m"]))
    with pytest.raises(ValueError, match="q2c_alpha"):
        call(q2c_alpha=None)
    with pytest.raises(ValueError, match="tasks"):
        call(tasks=("VR", "TVC"))
    with pytest.raises(ValueError, match="frames"):
        evalpass.VideoCorpus(torch.zeros(2, 513, 8), torch.ones(2, 513))
    big = evalpass.VideoCorpus(torch.randn(1100, 1, 8), torch.ones(1100, 1))
    with pytest.raises(ValueError, match="max_video"):
        evalpass.rank_modularized(big, torch.randn(2, 8), None, None, None, tasks=("VR",),
                                  max_video=1025)


# ------------------------------------------------------------------ HeroForVr
def _vr_and_vcmr(tmp_path):
    from hero_b200.model import VideoModelConfig
    from hero_b200.pretrain import HeroForVcmr, HeroForVr
    from tests.test_orchestration_cpu import _json
    fx, vx = gu.load("hier_tiny.npz"), gu.load("vsm_tiny.npz")
    d = gu.dims_of(fx)
    cfg = json.load(open(_json(tmp_path, d)))
    cfg["q_config"] = json.loads(str(vx["q_config"]))
    path = tmp_path / "vr.json"
    path.write_text(json.dumps(cfg))
    sd = {"v_encoder." + k: v for k, v in gu.weights_for(fx).items()}
    sd.update({k[5:]: torch.from_numpy(v) for k, v in vx.items() if k.startswith("head.")})
    kw = dict(vfeat_dim=d["vfeat_dim"], max_frm_seq_len=d["max_img_len"], lw_neg_ctx=8,
              lw_neg_q=8, margin=0.1)
    vr = HeroForVr(VideoModelConfig(str(path)), **kw)
    vcmr = HeroForVcmr(VideoModelConfig(str(path)), lw_st_ed=0, drop_svmr_prob=1.0, **kw)
    for mdl in (vr, vcmr):
        _, unexpected = mdl.load_state_dict(sd, strict=False)
        assert not unexpected
    vb, _ = gu.stored_batches(fx)

    def batch():
        b = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in vb.items()}
        for k in ("query_input_ids", "query_pos_ids", "query_attn_masks", "targets", "q_vidx"):
            b[k] = torch.from_numpy(vx[k])
        return b
    return vr.eval(), vcmr.eval(), batch, VideoModelConfig(str(path)), kw


def test_hero_for_vr_matches_vcmr_without_span_loss(tmp_path, monkeypatch):
    fake_rank_ops.install(monkeypatch)
    vr, vcmr, batch, _, _ = _vr_and_vcmr(tmp_path)
    assert vr.lw_st_ed == 0 and vr.drop_svmr_prob == 1.0
    assert set(vr.state_dict()) == set(vcmr.state_dict())
    with torch.no_grad():
        for task in ("msrvtt_video_sub", "msrvtt_video_only"):
            l_ctx, l_q = vr(batch(), task, compute_loss=True)
            _, r_ctx, r_q = vcmr(batch(), "tvr", compute_loss=True)
            assert torch.equal(l_ctx, r_ctx) and torch.equal(l_q, r_q)
            scores = vr(batch(), task, compute_loss=False)
            r_scores, st, ed = vcmr(batch(), "tvr", compute_loss=False)
            assert torch.equal(scores, r_scores) and st is None and ed is None
        with pytest.raises(ValueError, match="Unrecognized task"):
            vr(batch(), "tvr")
        b = batch()
        scores = vr.get_pred_from_raw_query(vr_frames := torch.randn(3, 5, 128), torch.ones(3, 5),
                                            b["query_input_ids"], b["query_pos_ids"],
                                            b["query_attn_masks"], cross=True)
        ref = vcmr.get_pred_from_raw_query(vr_frames, torch.ones(3, 5), b["query_input_ids"],
                                           b["query_pos_ids"], b["query_attn_masks"], cross=True)[0]
        assert torch.equal(scores, ref)


def test_hero_for_vr_requires_a_video_level_loss(tmp_path, monkeypatch):
    from hero_b200.pretrain import HeroForVr
    _, _, _, config, kw = _vr_and_vcmr(tmp_path)
    kw.update(lw_neg_ctx=0, lw_neg_q=0)
    with pytest.raises(AssertionError, match="lw_neg_ctx or lw_neg_q"):
        HeroForVr(config, **kw)
