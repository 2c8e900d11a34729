"""Full-corpus retrieval ranking on the GPU (hero_b200/csrc/rank.cu + evalpass): each kernel
against its torch fp32 restatement (tests/fake_rank_ops.py) at the TVR eval dimensions and on edge
shapes, deterministic tie order, the reference golden (tests/golden/vcmr_rank_tiny.npz) through
rank_modularized / full_vcmr_predictions, an end-to-end pass from embed_video_corpus, and the
absence of host synchronisation in rank_queries."""

import numpy as np
import pytest
import torch

from hero_b200 import evalpass, ops, synth
from tests import fake_rank_ops as ref
from tests import golden_util as gu
from tests.test_retrieval_cpu import (INTERVAL, _batches, _expected_eval_res, _golden,
                                      _rank_kw, _same_ranking, _same_records, _StubQueryModel)

pytestmark = pytest.mark.gpu
F32, I32 = torch.float32, torch.int32


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=F32, device="cuda")


def _neg(*shape):
    return torch.full(shape, -7, dtype=I32, device="cuda")


# ------------------------------------------------------------------ (a) kernels vs torch
@pytest.mark.parametrize("rows,n,k,apply_exp", [(80, 500, 100, True), (80, 500, 100, False),
                                                (3, 65536, 1024, False), (5, 7, 1, True),
                                                (4, 1000, 1000, False)])
def test_rank_topk_matches_torch(rows, n, k, apply_exp):
    g = torch.Generator().manual_seed(n + k)
    ld = n + 3
    x = torch.randn(rows, ld, generator=g).cuda()
    x[:, n:] = 1e9                                   # past n: must never be selected
    v, i = _nan(rows, k), _neg(rows, k)
    ops.rank_topk(x, n, k, v, i, alpha=20.0, apply_exp=apply_exp)
    rv, ri = torch.empty_like(v), torch.empty_like(i)
    ref.rank_topk(x, n, k, rv, ri, alpha=20.0, apply_exp=apply_exp)
    assert torch.equal(i, ri)
    if apply_exp:
        torch.testing.assert_close(v, rv, rtol=2e-6, atol=0)
    else:
        assert torch.equal(v, rv)


def _span_inputs(nv, L, d, n_pairs, seed, all_masked=(), one_frame=()):
    g = torch.Generator().manual_seed(seed)
    frames = torch.randn(nv, L, d, generator=g).cuda()
    lens = torch.randint(1, L + 1, (nv,), generator=g)
    lens[list(one_frame)] = 1
    mask = (torch.arange(L)[None] < lens[:, None]).to(torch.uint8)
    mask[list(all_masked)] = 0
    corpus = evalpass.VideoCorpus(frames, mask.cuda())
    nq = max(1, n_pairs // 7)
    p = torch.randn(nq, d, generator=g).cuda() * 0.05
    hi = torch.empty(nq, d, dtype=torch.bfloat16, device="cuda")
    lo, inv = torch.empty_like(hi), torch.empty(nq, dtype=F32, device="cuda")
    ops.l2norm_split(p, hi, lo, inv)
    s = torch.empty(nq, corpus.ld, dtype=F32, device="cuda")
    ops.gemm(hi, corpus.hi, s, a_lo=lo, b_lo=corpus.lo)
    rows = torch.randint(0, nq, (n_pairs,), generator=g).to(I32).cuda()
    clips = torch.randint(0, nv, (n_pairs,), generator=g)
    clips[:len(all_masked)] = torch.tensor(list(all_masked), dtype=torch.long)
    clips[len(all_masked):len(all_masked) + len(one_frame)] = torch.tensor(list(one_frame),
                                                                           dtype=torch.long)
    w = (torch.randn(2, 5, generator=g) * 0.3).cuda()
    return frames, corpus, p, s, inv, rows, clips.to(I32).cuda(), w


@pytest.mark.parametrize("nv,L", [(500, 100), (37, 13), (9, 1)])
def test_span_probs_match_torch(nv, L):
    d = 768
    frames, corpus, p, s, inv, rows, clips, w = _span_inputs(nv, L, d, 8000 if nv > 100 else 60,
                                                             seed=L, all_masked=(1, 2),
                                                             one_frame=(3,))
    st, ed = _nan(len(rows), L), _nan(len(rows), L)
    ops.vcmr_span_probs(s, rows, clips, inv, corpus.inv, corpus.mask, w[0].contiguous(),
                        w[1].contiguous(), nv, L, st, ed)
    # restatement from the raw (unnormalised) fp32 operands: p . c at every frame, masked or not
    sim = torch.einsum("bd,bld->bl", p[rows.long()], frames[clips.long()])
    rs, re = ref.span_probs_ref(sim, corpus.mask[clips.long()], w[0], w[1])
    assert not torch.isnan(st).any() and not torch.isnan(ed).any()
    torch.testing.assert_close(st, rs, rtol=3e-3, atol=2e-6)
    torch.testing.assert_close(ed, re, rtol=3e-3, atol=2e-6)


@pytest.mark.parametrize("nq,k,L,min_l,max_l,n,factor", [
    (80, 100, 55, 2, 16, 200, True),       # 44 400 B staged: below 48 KB, above 48 KB - static
    (7, 50, 100, 2, 16, 200, True),        # 40 200 B staged: the same window
    (80, 100, 100, 2, 16, 200, True),      # TVR eval config
    (6, 1, 100, 2, 16, 200, False),        # SVMR form
    (5, 3, 13, 1, 40, 1024, True),         # max_l > L, n above the candidate count
    (4, 2, 1, 0, 5, 10, True),             # 1-frame clips
    (3, 4, 7, 7, 9, 10, True),             # no valid span at all
])
def test_moment_topn_matches_torch(nq, k, L, min_l, max_l, n, factor):
    g = torch.Generator().manual_seed(nq * 31 + L)
    st = torch.softmax(torch.randn(nq, k, L, generator=g), -1).cuda()
    ed = torch.softmax(torch.randn(nq, k, L, generator=g), -1).cuda()
    st[:, 0, L // 2:] = 0.0                          # masked frames: probability 0
    vf = torch.exp(torch.rand(nq, k, generator=g) * 4).cuda() if factor else None
    score, jse = _nan(nq, n), _neg(nq, n, 3)
    ops.vcmr_moment_topn(st, ed, vf, nq, k, L, min_l, max_l, n, score, jse)
    rs, rj = ref.moment_topn_ref(st, ed, vf, L, min_l, max_l, n)
    assert torch.equal(jse, rj)
    assert torch.equal(score, rs)                    # same products in the same order


_FRESH_PROCESS = """
import sys, torch
sys.path.insert(0, sys.argv[1])
from hero_b200 import ops
from tests import fake_rank_ops as ref
g = torch.Generator().manual_seed(1)
nq, k, L, n = 8, 100, 55, 200
st = torch.softmax(torch.randn(nq, k, L, generator=g), -1).cuda()
ed = torch.softmax(torch.randn(nq, k, L, generator=g), -1).cuda()
vf = torch.rand(nq, k, generator=g).cuda()
score = torch.full((nq, n), float("nan"), device="cuda")
jse = torch.full((nq, n, 3), -7, dtype=torch.int32, device="cuda")
ops.vcmr_moment_topn(st, ed, vf, nq, k, L, 2, 16, n, score, jse)
rs, rj = ref.moment_topn_ref(st, ed, vf, L, 2, 16, n)
assert torch.equal(jse, rj) and torch.equal(score, rs)
print("ok")
"""


def test_moment_topn_first_launch_in_a_fresh_process():
    """The kernel's first launch in a process, with staged st / ed between 48 KB minus its static
    shared memory and 48 KB: it must not depend on an earlier, larger launch having raised the
    function's dynamic shared-memory limit."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _FRESH_PROCESS, root], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_moment_topn_stages_through_l2_when_large():
    """K * L too large for shared memory: st / ed are read from global memory."""
    nq, k, L = 2, 300, 100
    g = torch.Generator().manual_seed(5)
    st = torch.softmax(torch.randn(nq, k, L, generator=g), -1).cuda()
    ed = torch.softmax(torch.randn(nq, k, L, generator=g), -1).cuda()
    vf = torch.rand(nq, k, generator=g).cuda()
    score, jse = _nan(nq, 500), _neg(nq, 500, 3)
    ops.vcmr_moment_topn(st, ed, vf, nq, k, L, 2, 16, 500, score, jse)
    rs, rj = ref.moment_topn_ref(st, ed, vf, L, 2, 16, 500)
    assert torch.equal(jse, rj) and torch.equal(score, rs)


# ------------------------------------------------------------------ (b) ties, determinism
def test_exact_ties_come_out_in_index_order_and_runs_are_identical():
    x = torch.zeros(3, 3000, device="cuda")
    x[0, ::7] = 1.0                                  # 429 equal maxima, then 2571 equal zeros
    x[1] = torch.arange(3000, device="cuda").float().remainder(5)
    v, i = _nan(3, 1000), _neg(3, 1000)
    ops.rank_topk(x, 3000, 1000, v, i)
    assert i[0, :429].tolist() == list(range(0, 3000, 7))
    zeros = [c for c in range(3000) if c % 7][:1000 - 429]
    assert i[0, 429:].tolist() == zeros
    assert i[1, :600].tolist() == list(range(4, 3000, 5))
    assert i[2].tolist() == list(range(1000))
    st = torch.full((2, 3, 10), 0.1, device="cuda")
    ed = torch.full((2, 3, 10), 0.1, device="cuda")
    score, jse = _nan(2, 50), _neg(2, 50, 3)
    ops.vcmr_moment_topn(st, ed, None, 2, 3, 10, 1, 4, 50, score, jse)
    flat = (jse[..., 0] * 100 + jse[..., 1] * 10 + jse[..., 2]).tolist()
    assert all(f == sorted(f) for f in flat)
    fx, cfg = _golden()
    corpus = evalpass.VideoCorpus(torch.from_numpy(fx["frames"]).cuda(),
                                  torch.from_numpy(fx["c_attn_masks"]).cuda())
    args = (corpus, torch.from_numpy(fx["m"]).cuda(), torch.from_numpy(fx["p"]).cuda(),
            torch.from_numpy(fx["w_st"]).cuda(), torch.from_numpy(fx["w_ed"]).cuda())
    gt = torch.from_numpy(fx["gt_vidx"]).cuda()
    a = evalpass.rank_modularized(*args, gt_vidx=gt, **_rank_kw(cfg))
    b = evalpass.rank_modularized(*args, gt_vidx=gt, **_rank_kw(cfg))
    for t in a:
        for x1, x2 in zip(a[t], b[t]):
            assert torch.equal(x1, x2)


# ------------------------------------------------------------------ (c) reference golden
def test_golden_through_rank_modularized_and_full_vcmr_predictions():
    fx, cfg = _golden()
    corpus = evalpass.VideoCorpus(torch.from_numpy(fx["frames"]).cuda(),
                                  torch.from_numpy(fx["c_attn_masks"]).cuda())
    out = evalpass.rank_modularized(
        corpus, torch.from_numpy(fx["m"]).cuda(), torch.from_numpy(fx["p"]).cuda(),
        torch.from_numpy(fx["w_st"]).cuda(), torch.from_numpy(fx["w_ed"]).cuda(),
        gt_vidx=torch.from_numpy(fx["gt_vidx"]).cuda(), **_rank_kw(cfg))
    for q in range(len(fx["m"])):
        _same_ranking(out["VR"][0][q].cpu().numpy(), out["VR"][1][q].cpu().numpy(),
                      fx["vr_scores"][q], fx["vr_idx"][q])
        _same_ranking(out["VCMR"][0][q].cpu().numpy(), out["VCMR"][1][q].cpu().numpy(),
                      fx["vcmr_scores"][q], fx["vcmr_moments"][q])
        tri = fx["svmr_triples"][q]
        keys = np.stack([np.full(len(tri), fx["gt_vidx"][q]), tri[:, 0], tri[:, 1]], 1)
        _same_ranking(out["SVMR"][0][q].cpu().numpy(), out["SVMR"][1][q].cpu().numpy(),
                      tri[:, 2], keys.astype(np.int64))
    batches, video_ids, video2idx = _batches(fx)
    res = evalpass.full_vcmr_predictions(
        _StubQueryModel(fx).cuda(), corpus, batches, video_ids, video2idx,
        q2c_alpha=cfg["q2c_alpha"], max_vcmr_video=cfg["K"], min_pred_l=cfg["min_pred_l"],
        max_pred_l=cfg["max_pred_l"], max_before_nms=cfg["N"], vfeat_interval=INTERVAL)
    want = _expected_eval_res(fx, cfg, video_ids, video2idx)
    assert list(res) == ["SVMR", "VCMR", "VR", "video2idx"]
    for k in ("SVMR", "VCMR", "VR"):
        _same_records(res[k], want[k])


# ------------------------------------------------------------------ (d) end to end
def _cut_consistent(got_keys, got_vals, all_keys, all_vals, n, tol):
    """got == the restatement's top n, except that an entry may differ where the restatement's own
    score lies within tol of its n-th score."""
    order = np.argsort(-all_vals, kind="stable")
    cut = all_vals[order[min(n, len(order)) - 1]]
    top = {tuple(all_keys[o]) for o in order[:n]}
    val = {tuple(all_keys[o]): all_vals[o] for o in order}
    ref_sorted = all_vals[order[:n]]
    assert np.abs(np.asarray(got_vals) - ref_sorted[:len(got_vals)]).max() <= tol
    for k in map(tuple, got_keys):
        assert k in top or val[k] >= cut - tol, k
    for k in top - set(map(tuple, got_keys)):
        assert val[k] <= cut + tol, k


def test_end_to_end_from_embed_video_corpus(tmp_path):
    from hero_b200.evalpass import embed_video_corpus
    from tests.test_heads_cpu import _vcmr_model
    model, _, vx = _vcmr_model(tmp_path)
    model = model.cuda().eval()
    d = gu.dims_of(gu.load("hier_tiny.npz"))
    vbs = [synth.syn_tvr_ragged(batch_size=4, seed=70 + i, vfeat_dim=d["vfeat_dim"],
                                vocab=d["vocab"] - 7, t_range=t, s_range=(2, 4), l_range=(3, 8),
                                q_range=(3, 7))[0] for i, t in enumerate([(2, 9), (12, 20)])]
    emb, masks = embed_video_corpus(model, vbs, n_videos=8, max_clip_len=20)
    corpus = evalpass.VideoCorpus(emb, masks)
    nq = vx["query_input_ids"].shape[0]
    video_ids = [f"v{i}" for i in range(8)]
    video2idx = {v: i for i, v in enumerate(video_ids)}
    gt = [i % 8 for i in range(nq)]
    batch = dict(qids=list(range(nq)), vids=[video_ids[g] for g in gt],
                 targets=torch.zeros(nq, 2, dtype=torch.long),
                 query_input_ids=torch.from_numpy(vx["query_input_ids"]),
                 query_pos_ids=torch.from_numpy(vx["query_pos_ids"]),
                 query_attn_masks=torch.from_numpy(vx["query_attn_masks"]))
    K, N, alpha, lo, hi = 5, 40, 20.0, 1, 6
    res = evalpass.full_vcmr_predictions(model, corpus, [batch], video_ids, video2idx,
                                         q2c_alpha=alpha, max_vcmr_video=K, min_pred_l=lo,
                                         max_pred_l=hi, max_before_nms=N, vfeat_interval=1.0)
    # torch restatement of eval_vcmr.py:232-354 on the same embeddings
    with torch.no_grad():
        m = model.encode_txt_inputs(*(batch[k].cuda() for k in ("query_input_ids", "query_pos_ids",
                                                                "query_attn_masks")),
                                    attn_layer=model.q_feat_attn).float()
        c = emb.float()
        cos = torch.einsum("md,nld->mnl", torch.nn.functional.normalize(m, dim=-1, eps=1e-5),
                           torch.nn.functional.normalize(c, dim=-1, eps=1e-5))
        mk = masks.float()[None]
        s = (cos * mk + (1 - mk) * -1e4).max(-1).values
        f = torch.exp(alpha * s)
        p = model.video_query_linear(m)
        sim = torch.einsum("md,nld->mnl", p, c)
        L = c.shape[1]
        flat_sim = sim.reshape(-1, L)
        st, ed = ref.span_probs_ref(flat_sim, masks.to(torch.uint8).repeat(nq, 1),
                                    model.video_st_predictor.weight.reshape(-1),
                                    model.video_ed_predictor.weight.reshape(-1))
        st, ed = st.view(nq, 8, L), ed.view(nq, 8, L)
    band = ref.band_mask(L, lo, hi, "cuda").float()
    for q in range(nq):
        fq = f[q].cpu().numpy()
        tol_v = 5e-4 * float(np.abs(fq).max())   # exp(20 s) amplifies s's error
        got = res["VR"][q]["predictions"]
        _cut_consistent([(p_[0],) for p_ in got], [p_[3] for p_ in got],
                        np.arange(8)[:, None], fq, K, tol_v)
        prod = st[q][:, :, None] * f[q][:, None, None] * ed[q][:, None, :] * band
        idx = torch.nonzero(band.bool()[None].expand(8, L, L).reshape(-1)).flatten()
        keys = np.stack(np.unravel_index(idx.cpu().numpy(), (8, L, L)), 1)
        vals = prod.reshape(-1)[idx].cpu().numpy()
        tol = 5e-4 * float(np.abs(vals).max())
        # only moments inside the top-K clips are candidates: the restatement takes them from the
        # clips our VR list chose (equal to its own top K up to ties at the VR cut)
        chosen = {p_[0] for p_ in got}
        sel = np.array([k_[0] in chosen for k_ in keys])
        gm = res["VCMR"][q]["predictions"]
        _cut_consistent([(p_[0], int(p_[1]), int(p_[2]) - 1) for p_ in gm], [p_[3] for p_ in gm],
                        keys[sel], vals[sel], N, tol)
        g_ = gt[q]
        sv = (st[q, g_][:, None] * ed[q, g_][None, :] * band).reshape(-1)
        sidx = torch.nonzero(band.bool().reshape(-1)).flatten()
        skeys = np.stack([np.full(len(sidx), g_), *np.unravel_index(sidx.cpu().numpy(), (L, L))], 1)
        svals = sv[sidx].cpu().numpy()
        gs = res["SVMR"][q]["predictions"]
        _cut_consistent([(p_[0], int(p_[1]), int(p_[2]) - 1) for p_ in gs], [p_[3] for p_ in gs],
                        skeys, svals, N, 1e-4 * float(np.abs(svals).max()))


# ------------------------------------------------------------------ (e) no host sync
def test_rank_queries_does_not_synchronise(tmp_path):
    from hero_b200.loader import BatchStager
    from hero_b200.plan import PLAN_KEY, attach_plan
    from tests.test_heads_cpu import _vcmr_model
    model, _, vx = _vcmr_model(tmp_path)
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(3)
    corpus = evalpass.VideoCorpus(torch.randn(40, 24, 128, generator=g).cuda(),
                                  (torch.rand(40, 24, generator=g) > 0.2).cuda())
    qb = {k: torch.from_numpy(vx[k]) for k in ("query_input_ids", "query_pos_ids",
                                               "query_attn_masks")}
    tb = attach_plan({"input_ids": qb["query_input_ids"], "pos_ids": qb["query_pos_ids"],
                      "attn_masks": qb["query_attn_masks"]}, "txt")
    qb[PLAN_KEY] = tb[PLAN_KEY]
    qb["gt_vidx"] = torch.arange(len(vx["query_input_ids"]), dtype=I32)
    stager = BatchStager("cuda", depth=1)
    (dqb,), ready, _ = stager.stage(qb)
    torch.cuda.current_stream().wait_event(ready)
    kw = dict(q2c_alpha=20.0, max_video=10, min_pred_l=2, max_pred_l=16, max_before_nms=100,
              gt_vidx=dqb["gt_vidx"])
    evalpass.rank_queries(model, corpus, dqb, **kw)          # warm-up (allocations)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = evalpass.rank_queries(model, corpus, dqb, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert set(out) == {"VR", "VCMR", "SVMR"}
    assert not torch.isnan(out["VCMR"][0]).any()
