"""Video QA on the H100: the pooling kernels of csrc/qa.cu against torch autograd of the reference
expressions (model/videoQA.py:36-59), the query-fused embedding against torch, HeroForVideoQA
against the reference's outputs (tests/golden/videoqa_tiny.npz) and, at real dimensions, against
the reference module staged under oracle/_ref, a training step without host synchronisation, and
validate_videoqa."""
import json

import numpy as np
import pytest
import torch

from tests import fake_qa_ops
from tests import test_videoqa_cpu as cpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp(min=1e-12))


def _pool_case(nv, nq, length, H, lens, seed):
    """Packed rows with the frames of each (v, q) row first, a few extra (QA) rows between."""
    g = torch.Generator().manual_seed(seed)
    fmap = torch.full((nv * nq * length,), -1, dtype=torch.int32)
    nxt = 0
    for r in range(nv * nq):
        n = int(lens[r])
        fmap[r * length:r * length + n] = torch.arange(nxt, nxt + n, dtype=torch.int32)
        nxt += n + 3
    h = torch.randn(nxt + 1, H, generator=g)
    mask = (fmap >= 0).float()
    w_qa, w_st = torch.randn(1, H, generator=g) * 0.1, torch.randn(1, H, generator=g) * 0.1
    d_qa, d_st = torch.randn(nv * nq, H, generator=g), torch.randn(nv * length, H, generator=g)
    return [t.to(DEV) for t in (h, fmap, mask, w_qa, w_st, d_qa, d_st)]


@pytest.mark.parametrize("nv,nq,length,H,kind", [
    (4, 5, 100, 768, "tvqa"), (3, 4, 1, 64, "L1"), (3, 4, 9, 64, "one_frame"),
    (3, 1, 20, 128, "nq1"), (2, 5, 30, 96, "differ"), (2, 16, 512, 128, "max")])
def test_pool_kernels_match_torch_autograd(nv, nq, length, H, kind):
    from hero_b200 import functional as Fn
    g = torch.Generator().manual_seed(length + nq)
    if kind == "differ":           # masks differ between the candidates of a video
        lens = torch.randint(1, length + 1, (nv * nq,), generator=g)
    else:                          # the collate gives every candidate of a video the same clip
        lens = torch.randint(1, length + 1, (nv,), generator=g).repeat_interleave(nq)
        if kind == "one_frame":
            lens[:nq] = 1
    h, fmap, mask, w_qa, w_st, d_qa, d_st = _pool_case(nv, nq, length, H, lens, 3)
    # NaN-filled outputs: every element must be written
    from hero_b200 import ops
    a = torch.full((nv * nq * length,), float("nan"), device=DEV)
    b = torch.full_like(a, float("nan"))
    qa = torch.full((nv * nq, H), float("nan"), device=DEV)
    sp = torch.full((nv * length, H), float("nan"), device=DEV)
    ops.qa_pool_fwd(h, fmap, mask, w_qa.reshape(-1), w_st.reshape(-1), nv, nq, length, a, b, qa, sp)
    x = fake_qa_ops.padded(h, fmap, nv, nq, length).detach().requires_grad_(True)
    wq, ws = w_qa.clone().requires_grad_(True), w_st.clone().requires_grad_(True)
    sp_ref, qa_ref, a_ref, b_ref = fake_qa_ops.pool_ref(x, mask.view(nv, nq, length), wq, ws)
    for got, ref in ((qa, qa_ref.reshape(nv * nq, H)), (sp, sp_ref.reshape(nv * length, H)),
                     (a, a_ref), (b, b_ref)):
        assert torch.isfinite(got).all()
        torch.testing.assert_close(got, ref.detach(), rtol=1e-4, atol=1e-5)
    torch.autograd.backward([qa_ref.reshape(nv * nq, H), sp_ref.reshape(nv * length, H)],
                            [d_qa, d_st])
    hh = h.clone().requires_grad_(True)
    wq2, ws2 = w_qa.clone().requires_grad_(True), w_st.clone().requires_grad_(True)
    qa2, sp2 = Fn.qa_pool(hh, wq2, ws2, fmap, mask, nv, nq, length)
    torch.autograd.backward([qa2, sp2], [d_qa, d_st])
    keep = fmap.long() >= 0
    dh_ref = torch.zeros_like(h)
    dh_ref[fmap.long()[keep]] = x.grad.reshape(-1, H)[keep]
    torch.testing.assert_close(hh.grad, dh_ref, rtol=1e-4, atol=1e-5)
    assert _rel(wq2.grad, wq.grad) < 1e-4 and _rel(ws2.grad, ws.grad) < 1e-4
    # fixed-order reductions: bitwise reproducible
    wq3 = w_qa.clone().requires_grad_(True)
    qa3, sp3 = Fn.qa_pool(h, wq3, w_st, fmap, mask, nv, nq, length)
    torch.autograd.backward([qa3, sp3], [d_qa, d_st])
    assert torch.equal(wq3.grad, wq2.grad)


def test_pool_rejects_out_of_bounds_and_host_tensors():
    from hero_b200 import _lib, ops
    h, fmap, mask, w_qa, w_st, _, _ = _pool_case(1, 17, 2, 64, torch.ones(17), 0)
    out = torch.empty(64, device=DEV)
    with pytest.raises(ValueError):
        ops.qa_pool_fwd(h, fmap, mask, w_qa.reshape(-1), w_st.reshape(-1), 1, 17, 2, out, out, out,
                        out)
    with pytest.raises(_lib.HeroError):
        ops.qa_pool_fwd(h.cpu(), fmap, mask, w_qa.reshape(-1), w_st.reshape(-1), 1, 16, 2, out, out,
                        out, out)


def test_fused_embedding_forward_backward_match_torch(tmp_path):
    from hero_b200 import functional as Fn
    from hero_b200.plan import qa_plan
    vx = cpu.fixture()
    model = cpu.qa_model(tmp_path, vx).to(DEV)
    b = cpu.qa_batch(vx)
    qp = qa_plan(b)
    dev = qp.to(DEV)
    ce, te = model.v_encoder.c_encoder.embeddings, model.v_encoder.f_encoder.embeddings
    H = 128
    g = (torch.randn(qp.n_frm, H, generator=torch.Generator().manual_seed(0))).to(DEV)
    gb = g.to(torch.bfloat16).requires_grad_(True)
    cfg = {"drop": Fn.DropoutState(), "frm_p": 0.0, "qa_p": 0.0, "n_tok": qp.seq.n_tok, "n_frm": qp.n_frm, "n_qa": qp.n_qa,
           "frm_tok": dev.frm_tok, "frm_t": dev.frm_t, "qa_tok": dev.qa_tok, "qa_ids": dev.qa_ids,
           "qa_pos": dev.qa_pos, "cpos_off": dev.cpos_off, "cpos_idx": dev.cpos_idx,
           "qpos_off": dev.qpos_off, "qpos_idx": dev.qpos_idx, "pad_idx": te.padding_idx}
    params = [ce.position_embeddings.weight, ce.LayerNorm.weight, ce.LayerNorm.bias,
              te.word_embeddings.weight, te.position_embeddings.weight,
              te.token_type_embeddings.weight, te.LayerNorm.weight, te.LayerNorm.bias]
    emb, emb32 = Fn.qa_fused_embed(gb, cfg, params)
    # torch restatement (model/videoQA.py:68-78) on the packed rows
    ref = torch.empty(qp.seq.n_tok, H, device=DEV)
    gr = gb.detach().float().requires_grad_(True)
    fr = ce.LayerNorm(gr + ce.position_embeddings.weight[dev.frm_t.long()])
    qr = te.LayerNorm(te.word_embeddings.weight[dev.qa_ids.long()]
                      + te.position_embeddings.weight[dev.qa_pos.long()]
                      + te.token_type_embeddings.weight[1])
    ref = ref.index_put((dev.frm_tok.long(),), fr).index_put((dev.qa_tok.long(),), qr)
    torch.testing.assert_close(emb32, ref.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(emb.float(), ref.detach(), rtol=1e-2, atol=1e-2)
    dy = torch.randn(qp.seq.n_tok, H, device=DEV).to(torch.bfloat16)
    grads = torch.autograd.grad(emb, [gb] + params, dy)
    refs = torch.autograd.grad(ref, [gr] + params, dy.float())
    for got, want in zip(grads, refs):
        assert _rel(got, want) < 1e-2


def test_model_matches_reference_fixture(tmp_path):
    vx = cpu.fixture()
    model = cpu.qa_model(tmp_path, vx).to(DEV)

    def batch():
        return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in cpu.qa_batch(vx).items()}

    with torch.no_grad():
        for task in ("tvqa", "how2qa"):
            logits = model(batch(), task, compute_loss=False).cpu().numpy()
            qa_loss, t_loss = model(batch(), task)
            ref = vx[f"{task}.logits"]
            assert np.abs(logits - ref).max() <= 2e-2 * max(np.abs(ref).max(), 1.0)
            assert abs(float(qa_loss) - float(vx[f"{task}.qa_loss"])) < 2e-2
            assert abs(float(t_loss) - float(vx[f"{task}.temporal_loss"])) < 2e-2
    lw = json.loads(str(vx["config"]))["lw_st_ed"]
    qa_loss, t_loss = model(batch(), "tvqa")
    (qa_loss + lw * t_loss).backward()
    params = dict(model.named_parameters())
    for name in json.loads(str(vx["grad_params"])):
        rel = _rel(params[name].grad.cpu(), torch.from_numpy(vx["g." + name]))
        assert rel < 3e-2, (name, rel)


def _tvqa_model(seed=0):
    import tempfile
    from hero_b200.model import VideoModelConfig
    from hero_b200.videoqa import HeroForVideoQA
    from oracle import gen_golden as gg
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(gg.model_json(768, 3072, 12, 6, 3, 50272), f)
        path = f.name
    torch.manual_seed(seed)
    return HeroForVideoQA(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100), path


def test_training_step_does_not_sync_with_the_host():
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    model, _ = _tvqa_model()
    model = model.to(DEV).train()
    b = attach_plan(synth.syn_tvqa(seed=5), kind="videoqa")
    b = synth.to_device(b, DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        qa_loss, t_loss = model(b, "tvqa")
        (qa_loss + 0.4 * t_loss).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(qa_loss) and torch.isfinite(t_loss)
    for mod in (model.qa_pool, model.qa_pred_head, model.st_ed_pool, model.st_ed_pred_head):
        for n, p in mod.named_parameters():
            if n in ("LayerNorm.bias", "linear_2.bias"):     # zero: softmax shift invariance
                continue
            assert p.grad is not None and float(p.grad.abs().sum()) > 0, n


def test_validate_videoqa_on_synthetic_batches():
    from hero_b200 import evalpass, synth
    from hero_b200.plan import attach_plan
    model, _ = _tvqa_model()
    model = model.to(DEV)
    loader = []
    for s in (1, 2):
        b = attach_plan(synth.syn_videoqa_batch(n_videos=3, n_cand=5, seed=s), kind="videoqa")
        b = synth.to_device(b, DEV)
        b["qids"] = [10 * s + i for i in range(3)]
        loader.append(b)
    copies = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(t, *a, **k):
        copies.append(tuple(t.shape))
        return real_cpu(t, *a, **k)

    torch.cuda.set_sync_debug_mode("warn")
    try:
        torch.Tensor.cpu = counting_cpu
        val_log, results, logits = evalpass.validate_videoqa(model, loader, "val")
    finally:
        torch.Tensor.cpu = real_cpu
        torch.cuda.set_sync_debug_mode("default")
    assert len(copies) == 2
    assert set(results) == {"10", "11", "12", "20", "21", "22"}
    assert set(val_log) == {"valid/loss", "valid/acc", "valid/ex_per_s"}
    assert np.isfinite(val_log["valid/loss"])


def _reference_module():
    from oracle import gen_golden as gg
    from oracle import stage_ref
    ref = stage_ref.available()
    if ref is None:
        pytest.skip("no staged reference under oracle/_ref")
    gg.REF = ref
    gg.install_stubs()
    from model.model import VideoModelConfig
    from model.videoQA import HeroForVideoQA
    return VideoModelConfig, HeroForVideoQA


# Gradients of the two pooling weights: their size depends on how far the candidates of one video
# differ, which is little at a random initialisation. They are measured against the reference's own
# bf16-autocast run (SURVEY §8c yardstick: <= 1.5x its error); every other gradient <= 3e-2.
YARDSTICK_GRADS = ("qa_pool.weight", "st_ed_pool.weight")
ZERO_GRADS = ("qa_pred_head.LayerNorm.bias", "qa_pred_head.linear_2.bias",
              "st_ed_pred_head.LayerNorm.bias", "st_ed_pred_head.linear_2.bias")


def test_real_dimensions_match_staged_reference():
    """6 + 3 layers, H 768, TVQA preset: logits, losses, head and encoder gradients against the
    reference's HeroForVideoQA in fp32 on the same GPU (SURVEY §8c bounds), with the same reference
    under torch bf16 autocast as the yardstick."""
    VideoModelConfig, RefQA = _reference_module()
    from hero_b200 import synth
    model, path = _tvqa_model(seed=3)
    ref = RefQA(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(model.state_dict())
    model, ref = model.to(DEV).eval(), ref.to(DEV).eval()
    hb = synth.syn_tvqa(seed=9)
    outs = []
    for m, bf16 in ((model, False), (ref, False), (ref, True)):
        m.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
            logits = m(dict(synth.to_device(hb, DEV)), "tvqa", compute_loss=False)
            qa_loss, t_loss = m(dict(synth.to_device(hb, DEV)), "tvqa")
        (qa_loss + 0.4 * t_loss).backward()
        outs.append((logits.detach().float(), qa_loss.detach().float(), t_loss.detach().float(),
                     {n: p.grad.detach().clone() for n, p in m.named_parameters()
                      if p.grad is not None}))
    (lo, qo, to, go), (lr, qr, tr, gr), (_, _, _, gb) = outs
    assert float((lo - lr).abs().max()) <= 2e-2 * max(float(lr.abs().max()), 1.0)
    assert abs(float(qo) - float(qr)) < 2e-2 and abs(float(to) - float(tr)) < 2e-2
    heads = [n for n in gr if n.startswith(("qa_pool", "st_ed_pool", "qa_pred_head",
                                            "st_ed_pred_head")) and n not in ZERO_GRADS]
    names = heads + [
        "v_encoder.c_encoder.encoder.layer.0.attention.self.query.weight",
        "v_encoder.c_encoder.encoder.layer.0.attention.self.value.weight",
        "v_encoder.c_encoder.encoder.layer.2.output.dense.weight",
        "v_encoder.c_encoder.embeddings.position_embeddings.weight",
        "v_encoder.f_encoder.embeddings.word_embeddings.weight",
        "v_encoder.f_encoder.encoder.layer.0.output.dense.weight"]
    rel = {n: (_rel(go[n], gr[n]), _rel(gb[n], gr[n])) for n in names}
    for n, (ours, bf16) in rel.items():
        print(f"grad rel err vs fp32 reference: {n}: ours {ours:.4f}, reference bf16 {bf16:.4f}")
    for n, (ours, bf16) in rel.items():
        if n in YARDSTICK_GRADS:
            assert ours <= 1.5 * bf16, (n, ours, bf16)
        else:
            assert ours < 3e-2, (n, ours, bf16)


def test_prefetch_loader_stages_the_query_fused_plan():
    """PrefetchLoader builds (in-process fallback) or takes (collate-attached) both video QA plans
    and uploads the QaPlan through the stager's buffers; the step then makes no host sync."""
    from hero_b200 import synth
    from hero_b200.loader import PrefetchLoader
    from hero_b200.plan import PLAN_KEY, QA_PLAN_KEY, attach_plan
    model, _ = _tvqa_model()
    model = model.to(DEV).train()
    host = [synth.syn_videoqa_batch(n_videos=2, n_cand=5, seed=s) for s in (3, 4)]
    host[1] = attach_plan(host[1], kind="videoqa")
    n = 0
    for b in PrefetchLoader(host, device=DEV, depth=2):
        assert b[PLAN_KEY] is not None and b[QA_PLAN_KEY] is not None
        assert b[QA_PLAN_KEY].dev is not None
        torch.cuda.set_sync_debug_mode("error")
        try:
            qa_loss, t_loss = model(b, "tvqa")
            (qa_loss + 0.4 * t_loss).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.isfinite(qa_loss) and torch.isfinite(t_loss)
        n += 1
    assert n == 2
