"""Host-side packing plans (pure numpy): checked against the padded-layout semantics of the
reference as restated by the oracle (gather of cat[img, txt]; collect_frame_outputs)."""
import numpy as np
import pytest
import torch

from hero_b200 import synth
from hero_b200.plan import FPlan, ReprPlan, SeqPlan, TxtPlan, plan_inputs
from oracle import hero_oracle as orc


def _ragged(seed=3, bs=4):
    return synth.syn_tvr_ragged(batch_size=bs, seed=seed, vfeat_dim=8, vocab=60, t_range=(6, 14),
                                s_range=(2, 5), l_range=(3, 9), q_range=(3, 8))


def test_seqplan_roundtrip():
    mask = np.array([[1, 1, 0, 0], [0, 1, 1, 1], [0, 0, 0, 0], [1, 0, 1, 0]])
    sp = SeqPlan(mask)
    assert sp.n_tok == 7 and sp.max_len == 3
    assert sp.cu.tolist() == [0, 2, 5, 5, 7]
    assert sp.tok_flat.tolist() == [0, 1, 5, 6, 7, 12, 14]
    assert sp.pad_to_tok[sp.tok_flat].tolist() == list(range(7))
    assert (sp.pad_to_tok >= 0).sum() == 7


def test_fplan_matches_gather_of_cat_img_txt():
    vb, _ = _ragged()
    R, max_vl = vb["f_v_feats"].shape[:2]
    max_sl = vb["f_sub_input_ids"].shape[1]
    fp = FPlan(vb["f_attn_masks"], vb["f_gather_index"], max_vl, max_sl)
    img_id = torch.arange(R * max_vl).view(R, max_vl)                 # unique id per frame slot
    txt_id = 10_000 + torch.arange(R * max_sl).view(R, max_sl)         # unique id per text slot
    ref = torch.gather(torch.cat([img_id, txt_id], 1), 1, vb["f_gather_index"])
    packed = np.full(fp.seq.n_tok, -1, np.int64)
    packed[fp.img_tok] = img_id.view(-1).numpy()[fp.img_src]
    packed[fp.txt_tok] = txt_id.view(-1).numpy()[fp.txt_src]
    valid = vb["f_attn_masks"].bool().numpy()
    assert np.array_equal(packed, ref.numpy()[valid])
    assert fp.n_img + fp.n_txt == fp.seq.n_tok == int(valid.sum())
    # zero-frame subtitles contribute no image token (their dummy frame is masked)
    assert fp.n_img == sum(len(fr) for clip in vb["sub_idx2frame_idx"] for _, fr in clip)


def test_cplan_equals_collect_frame_outputs_and_its_transpose():
    vb, _ = _ragged(seed=9, bs=5)
    plan = ReprPlan(vb)
    R, n = vb["f_attn_masks"].shape
    B, T = vb["c_attn_masks"].shape
    H = 6
    g = torch.Generator().manual_seed(0)
    f_out = torch.randn(R, n, H, generator=g)
    ref = orc.collect_frame_outputs((B, T, H), f_out, vb["num_subs"], vb["sub_idx2frame_idx"])
    f_packed = f_out.view(-1, H).numpy()[plan.f.seq.tok_flat]
    c = plan.c
    got = np.zeros((c.seq.n_tok, H), np.float32)
    for i in range(c.seq.n_tok):
        for e in range(c.fwd_off[i], c.fwd_off[i + 1]):
            got[i] += f_packed[c.fwd_idx[e]]
    assert np.allclose(got, ref.view(-1, H).numpy()[c.seq.tok_flat], atol=1e-6)
    # adjoint: <A f, y> == <f, A^T y>
    y = torch.randn(c.seq.n_tok, H, generator=g).numpy()
    aty = np.zeros((plan.f.seq.n_tok, H), np.float32)
    for i in range(plan.f.seq.n_tok):
        for e in range(c.bwd_off[i], c.bwd_off[i + 1]):
            aty[i] += y[c.bwd_idx[e]]
    assert np.isclose((got * y).sum(), (f_packed * aty).sum(), rtol=1e-4)


def test_duplicate_frame_assignments_accumulate():
    """model/model.py:182-184 accumulates when a frame is listed under two subtitles."""
    gen = torch.Generator().manual_seed(1)
    clip = synth.make_clip(gen, 6, [[0, 1, 2], [2, 3]], [3, 4], vfeat_dim=8, vocab=50)
    vb = synth.video_batch([clip])
    plan = ReprPlan(vb)
    c = plan.c
    counts = np.diff(c.fwd_off)
    assert counts.tolist() == [1, 1, 2, 1, 0, 0]


def _check_pos_csr(e, name, n):
    """The position-table CSR lists every packed token once, under the position id it reads."""
    pos, off, idx = e[name + "_pos"], e[name + "pos_off"], e[name + "pos_idx"]
    assert off[-1] == n == pos.size and np.array_equal(np.sort(idx), np.arange(n))
    for p in range(len(off) - 1):
        assert (pos[idx[off[p]:off[p + 1]]] == p).all()


def test_txt_plan_and_table_csr():
    _, qb = _ragged()
    tp = TxtPlan(**plan_inputs(qb, "txt"))
    valid = qb["attn_masks"].bool().numpy()
    assert tp.f.n_img == 0 and tp.f.n_txt == int(valid.sum())
    ids = qb["input_ids"].view(-1).numpy()[tp.f.txt_src]
    assert np.array_equal(ids, qb["input_ids"].numpy()[valid])
    e = tp.f.emb
    assert np.array_equal(e["txt_ids"], ids)
    pos = np.broadcast_to(qb["pos_ids"].numpy(), valid.shape)[valid]
    assert np.array_equal(e["txt_pos"], pos)
    _check_pos_csr(e, "txt", tp.f.n_txt)
    # without position ids: SubEmbeddings.create_position_ids_from_input_ids, on the host
    from types import SimpleNamespace
    from hero_b200.embed import SubEmbeddings
    tp2 = TxtPlan(**dict(plan_inputs(qb, "txt"), pos_ids=None))
    want = SubEmbeddings.create_position_ids_from_input_ids(SimpleNamespace(padding_idx=1),
                                                            qb["input_ids"])
    assert np.array_equal(tp2.f.emb["txt_pos"], want.numpy()[valid])
    _check_pos_csr(tp2.f.emb, "txt", tp2.f.n_txt)


def test_dense_canonical_batch_shapes():
    vb, qb = synth.syn_tvr_dense(batch_size=2, vfeat_dim=16)
    assert tuple(vb["f_sub_input_ids"].shape) == (40, 20)
    assert tuple(vb["f_v_feats"].shape) == (40, 5, 16)
    assert tuple(vb["f_attn_masks"].shape) == (40, 25)
    assert tuple(vb["c_v_feats"].shape) == (2, 100, 16)
    plan = ReprPlan(vb)
    assert plan.f.seq.n_tok == 40 * 25 and plan.c.seq.n_tok == 200
    assert plan.c.n_pairs == 200 and plan.f.seq.max_len == 25 and plan.c.seq.max_len == 100


def test_plan_pool_builds_the_same_plans_in_worker_processes():
    """PlanPool (collate-side plan building in worker processes) == attach_plan in-process, and
    the JointPlan of the fused video+query pass arrives prebuilt."""
    from hero_b200.plan import PLAN_KEY, JointPlan, PlanPool, attach_plan
    vb, qb = synth.syn_tvr_ragged(batch_size=3, seed=5, t_range=(10, 20), s_range=(2, 4),
                                  l_range=(4, 10))
    pool = PlanPool(workers=1)
    try:
        fut = pool.submit(vb, qb)
        vb2, qb2 = PlanPool.attach(fut, dict(vb), dict(qb))
    finally:
        pool.shutdown()
    ref_v = attach_plan(dict(vb))[PLAN_KEY]
    ref_q = attach_plan(dict(qb), kind="txt")[PLAN_KEY]
    got_v, got_q = vb2[PLAN_KEY], qb2[PLAN_KEY]
    for a, b in ((got_v.f.arrays("f_"), ref_v.f.arrays("f_")),
                 (got_v.c.arrays("c_"), ref_v.c.arrays("c_")),
                 (got_q.f.arrays("f_"), ref_q.f.arrays("f_")),
                 (got_v.__dict__["_joint"].arr, JointPlan(ref_v, ref_q).arr)):
        assert a.keys() == b.keys()
        for k in a:
            assert np.array_equal(a[k], b[k]), k
    assert got_v.__dict__["_joint"].t is got_q


def test_prefetch_loader_attaches_plans_in_order_without_cuda():
    """hero_b200.loader.PrefetchLoader._with_plans (the host half of the loader): batches come out
    in order, a plan attached by the collate function is kept, a missing one is built (here in
    process), single dicts and (video, query) pairs are both accepted."""
    from hero_b200.loader import PrefetchLoader
    from hero_b200.plan import PLAN_KEY, attach_plan
    items = []
    for seed in range(4):
        vb, qb = synth.syn_tvr_ragged(batch_size=2, seed=40 + seed, t_range=(8, 12),
                                      s_range=(2, 3), l_range=(3, 6))
        vb["_tag"] = seed
        items.append((vb, qb) if seed % 2 == 0 else vb)
    pre = attach_plan(dict(items[1]))[PLAN_KEY]
    items[1][PLAN_KEY] = pre
    ld = PrefetchLoader.__new__(PrefetchLoader)
    ld.pool = None
    out = list(ld._with_plans(iter(items)))
    assert [(b[0] if isinstance(b, tuple) else b)["_tag"] for b in out] == [0, 1, 2, 3]
    assert isinstance(out[0], tuple) and not isinstance(out[1], tuple)
    assert out[1][PLAN_KEY] is pre
    for b in out:
        vb = b[0] if isinstance(b, tuple) else b
        assert vb[PLAN_KEY] is not None
        if isinstance(b, tuple):
            assert b[1][PLAN_KEY] is not None
    assert PLAN_KEY not in items[0][0]          # the loader works on copies of the dicts


def test_frame_slots_map_back_to_clip_frames():
    """ReprPlan.f.img_src_c: every packed frame token of the subtitle rows points at the clip frame
    it was copied from (data/data.py fills f_v_feats with index_select(c_v_feats, frames)), so a
    batch may drop `f_v_feats`; without it max_vl comes from f_v_pos_ids."""
    vb, _ = synth.syn_tvr_ragged(batch_size=4, seed=61, t_range=(9, 15), s_range=(2, 5),
                                 l_range=(3, 7))
    plan = ReprPlan(vb)
    D = vb["c_v_feats"].shape[-1]
    from_f = vb["f_v_feats"].reshape(-1, D)[torch.from_numpy(plan.f.img_src).long()]
    from_c = vb["c_v_feats"].reshape(-1, D)[torch.from_numpy(plan.f.img_src_c).long()]
    assert plan.f.n_img > 0 and (plan.f.img_src_c >= 0).all()
    assert torch.equal(from_f, from_c)
    slim = {k: v for k, v in vb.items() if k != "f_v_feats"}
    plan2 = ReprPlan(slim)
    assert plan2.f.max_vl == plan.f.max_vl
    assert np.array_equal(plan2.f.img_src_c, plan.f.img_src_c)


def test_plan_invariants_and_position_csrs_on_random_batches():
    """Property test (hypothesis): for random ragged batches — including subtitles without frames,
    frames matched by no subtitle or by several, single-token rows — the plan is a bijection
    between packed tokens and valid padded positions, attention tiles partition the token stream
    without splitting a sequence, the two frame-merge CSRs are transposes of each other, the
    joint (video + query) plan is the concatenation of its parts, and every position-table CSR
    lists each token under the position id it reads."""
    from hypothesis import given, settings, strategies as st
    from hero_b200.plan import ATTN_TILE, JointPlan

    @settings(max_examples=25, deadline=None)
    @given(st.integers(0, 10_000), st.integers(1, 5))
    def check(seed, bs):
        vb, qb = synth.syn_tvr_ragged(batch_size=bs, seed=seed, vfeat_dim=8, vocab=60,
                                      t_range=(3, 40), s_range=(1, 6), l_range=(1, 9),
                                      q_range=(1, 8))
        rp, tp = ReprPlan(vb), TxtPlan(**plan_inputs(qb, "txt"))
        for sp, mask in ((rp.f.seq, vb["f_attn_masks"]), (rp.c.seq, vb["c_attn_masks"]),
                         (tp.f.seq, qb["attn_masks"])):
            valid = np.flatnonzero(mask.numpy().reshape(-1))
            assert np.array_equal(np.sort(sp.tok_flat), valid)            # bijection
            assert np.array_equal(sp.pad_to_tok[sp.tok_flat], np.arange(sp.n_tok))
            assert sp.tile_ntok.sum() == sp.n_tok and (sp.tile_ntok <= ATTN_TILE).all()
            assert np.array_equal(sp.tile_tok0, np.concatenate([[0], np.cumsum(sp.tile_ntok)[:-1]]))
            starts = set(sp.cu[:-1].tolist()) | {sp.n_tok}
            assert all(int(t) in starts for t in sp.tile_tok0)            # tiles start at sequences
            assert ((sp.seq_hi - sp.seq_lo) == np.repeat(sp.lens, sp.lens)).all()
        c = rp.c
        fwd = {(int(i), int(c.fwd_idx[e])) for i in range(c.seq.n_tok)
               for e in range(c.fwd_off[i], c.fwd_off[i + 1])}
        bwd = {(int(c.bwd_idx[e]), int(j)) for j in range(rp.f.seq.n_tok)
               for e in range(c.bwd_off[j], c.bwd_off[j + 1])}
        assert fwd == bwd and len(fwd) == c.n_pairs
        assert (rp.f.img_src_c >= 0).all()
        jp = JointPlan(rp, tp)
        a = rp.f.seq.n_tok
        assert jp.n_tok == a + tp.f.seq.n_tok and jp.n_tiles == rp.f.seq.n_tiles + tp.f.seq.n_tiles
        assert np.array_equal(jp.arr["j_seq_lo"][a:], tp.f.seq.seq_lo + a)
        for e, n in ((rp.f.emb, rp.f.n_txt), (tp.f.emb, tp.f.n_txt), (jp.arr, jp.n_txt)):
            _check_pos_csr(e, "txt", n)
        _check_pos_csr(rp.f.emb, "img", rp.f.n_img)
        assert np.array_equal(jp.arr["txt_pos"], np.concatenate([rp.f.emb["txt_pos"],
                                                                 tp.f.emb["txt_pos"]]))
        # a query plan without token ids cannot feed the joint embedding
        with pytest.raises(ValueError, match="input_ids"):
            JointPlan(rp, TxtPlan(qb["attn_masks"], pos_ids=qb["pos_ids"]))

    check()


def test_long_rows_become_trailing_tiles_and_joint_plans_keep_them_last():
    """Rows of more than 128 valid tokens (max_txt_len + matched frames; the position table allows
    514) are single-sequence tiles at the END of the tile list — also after concatenating the
    video rows' and the query rows' plans."""
    import numpy as np
    from hero_b200.plan import ATTN_LONG_MAX, SeqPlan

    def mask_of(lens):
        m = np.zeros((len(lens), max(lens)), np.int64)
        for r, n in enumerate(lens):
            m[r, :n] = 1
        return m

    lens = [30, 200, 5, 128, 129, 60, 70]
    sp = SeqPlan(mask_of(lens))
    assert sp.n_long == 2 and sp.max_long == 200
    n_short = sp.n_tiles - sp.n_long
    assert sp.tile_ntok[n_short:].tolist() == [200, 129]
    assert all(n <= 128 for n in sp.tile_ntok[:n_short])
    # every token is covered exactly once and no tile splits a sequence
    cover = np.zeros(sp.n_tok, np.int64)
    for a, n in zip(sp.tile_tok0, sp.tile_ntok):
        cover[a:a + n] += 1
        assert a in set(sp.cu.tolist()) and a + n in set(sp.cu.tolist())
    assert (cover == 1).all()
    assert sp.tile_tok0[n_short:].tolist() == [30, 30 + 200 + 5 + 128]
    import pytest
    with pytest.raises(ValueError, match="row 1"):
        SeqPlan(mask_of([3, ATTN_LONG_MAX + 1]))


def test_tiles_hold_at_most_16_sequences():
    """The attention kernels apply the block-diagonal mask as a K = 16 membership MMA
    (csrc/attention_tc.cu): a tile closes after 128 tokens OR 16 sequences, whichever comes first,
    including across empty rows, long rows and the joint (video + query) concatenation."""
    import numpy as np
    from hero_b200.plan import ATTN_TILE_SEQS, SeqPlan

    rng = np.random.RandomState(3)
    for _ in range(20):
        lens = rng.choice([0, 1, 2, 3, 5, 9, 40, 130], size=rng.randint(1, 120)).tolist()
        if max(lens) == 0:
            lens[0] = 1
        m = np.zeros((len(lens), max(lens)), np.int64)
        for r, n in enumerate(lens):
            m[r, :n] = 1
        sp = SeqPlan(m)
        starts = np.asarray([c for c, n in zip(sp.cu[:-1], np.diff(sp.cu)) if n > 0])
        len_at = {int(c): int(n) for c, n in zip(sp.cu[:-1], np.diff(sp.cu)) if n > 0}
        n_short = sp.n_tiles - sp.n_long
        assert int(sp.tile_ntok.sum()) == sp.n_tok
        for a, n in zip(sp.tile_tok0[:n_short], sp.tile_ntok[:n_short]):
            assert 0 < n <= 128
            assert ((starts >= a) & (starts < a + n)).sum() <= ATTN_TILE_SEQS
        # tiles are maximal: merging two neighbours would break one of the two limits
        for (a, n), (b, k) in zip(zip(sp.short_tok0, sp.short_ntok),
                                  zip(sp.short_tok0[1:], sp.short_ntok[1:])):
            if a + n == b:      # adjacent in the token stream (no long row between them)
                both = ((starts >= a) & (starts < b + k)).sum()
                first_of_next = len_at[int(b)]
                assert n + first_of_next > 128 or \
                    ((starts >= a) & (starts < a + n)).sum() == ATTN_TILE_SEQS, (a, n, b, k, both)


def test_zero_grads_async_on_cpu_is_a_plain_zero(monkeypatch):
    import torch
    from hero_b200.params import flat_of
    from tests import fake_ops
    fake_ops.install(monkeypatch)      # CPU process: the bf16 mirror cast has no CUDA library

    lin = torch.nn.Linear(4, 3)
    fp = flat_of(lin, torch.device("cpu"))
    g = fp.ensure_flat_grads()
    g.fill_(2.0)
    fp.zero_grads_async()
    fp.wait_grads_zeroed()
    assert float(g.abs().sum()) == 0.0
    assert float(lin.weight.grad.abs().sum()) == 0.0
