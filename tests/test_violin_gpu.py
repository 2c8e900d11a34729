"""VIOLIN on the H100: the single-pooling mode of the csrc/qa.cu kernels against torch autograd of
the reference expression (model/violin.py:30-47) and against the two-pooling call, HeroForViolin
against the reference's outputs (tests/golden/violin_tiny.npz) and, at real dimensions, against
the reference module staged under oracle/_ref, a training step without host synchronisation,
validate_violin, and PrefetchLoader transport of the VIOLIN plans."""
import json

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from tests import fake_qa_ops, fake_violin_ops
from tests import test_videoqa_gpu as qa_gpu
from tests import test_violin_cpu as cpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
_rel = qa_gpu._rel


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


@pytest.mark.parametrize("rows,length,kind", [
    (8, 100, "violin"), (6, 1, "L1"), (5, 9, "one_frame"), (4, 512, "max")])
def test_single_pool_kernels_match_torch_autograd(rows, length, kind):
    from hero_b200 import functional as Fn
    from hero_b200 import ops
    H = 768
    g = torch.Generator().manual_seed(length + rows)
    lens = torch.randint(1, length + 1, (rows,), generator=g)
    if kind == "one_frame":
        lens[:2] = 1
    if kind == "max":
        lens[0] = length
    h, fmap, mask, w, w_st, d_pool, _ = qa_gpu._pool_case(rows, 1, length, H, lens, 5)
    wv = w.reshape(-1)
    # NaN-filled outputs: every element must be written
    a, pooled = _nan(rows * length), _nan(rows, H)
    ops.qa_pool_fwd(h, fmap, mask, wv, None, rows, 1, length, a, None, pooled, None)
    x = fake_qa_ops.padded(h, fmap, rows, 1, length).view(rows, length, H)
    x = x.detach().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    pooled_ref, a_ref = fake_violin_ops.pool_ref(x, mask.view(rows, length), wr)
    for got, ref in ((pooled, pooled_ref), (a, a_ref)):
        assert torch.isfinite(got).all()
        torch.testing.assert_close(got, ref.detach(), rtol=1e-4, atol=1e-5)
    # the single pooling computes exactly the softmax-over-l half of the two-pooling call
    a2, b2 = _nan(rows * length), _nan(rows * length)
    qa2, sp2 = _nan(rows, H), _nan(rows * length, H)
    ops.qa_pool_fwd(h, fmap, mask, wv, w_st.reshape(-1), rows, 1, length, a2, b2, qa2, sp2)
    assert torch.equal(a, a2) and torch.equal(pooled, qa2)
    # backward against autograd
    pooled_ref.backward(d_pool)
    hh = h.clone().requires_grad_(True)
    w1 = w.clone().requires_grad_(True)
    out = Fn.qa_pool(hh, w1, None, fmap, mask, rows, 1, length)
    assert torch.is_tensor(out) and out.shape == (rows, H)
    out.backward(d_pool)
    keep = fmap.long() >= 0
    dh_ref = torch.zeros_like(h)
    dh_ref[fmap.long()[keep]] = x.grad.reshape(-1, H)[keep]
    torch.testing.assert_close(hh.grad, dh_ref, rtol=1e-4, atol=1e-5)
    assert _rel(w1.grad, wr.grad) < 1e-4
    # fixed-order reductions: bitwise reproducible
    w2 = w.clone().requires_grad_(True)
    Fn.qa_pool(h, w2, None, fmap, mask, rows, 1, length).backward(d_pool)
    assert torch.equal(w2.grad, w1.grad)


def test_single_pool_rejects_a_mix_of_null_and_set_st_arguments():
    from hero_b200 import _lib, ops
    rows, length, H = 2, 4, 64
    h, fmap, mask, w, w_st, d_pool, _ = qa_gpu._pool_case(rows, 1, length, H, torch.ones(rows), 0)
    a, b = torch.empty(rows * length, device=DEV), torch.empty(rows * length, device=DEV)
    pooled, sp = torch.empty(rows, H, device=DEV), torch.empty(rows * length, H, device=DEV)
    wv, sv = w.reshape(-1), w_st.reshape(-1)
    for args in ((None, b, sp), (None, b, None), (None, None, sp), (sv, None, sp), (sv, b, None)):
        ws, bb, ss = args
        with pytest.raises(_lib.HeroError):
            ops.qa_pool_fwd(h, fmap, mask, wv, ws, rows, 1, length, a, bb, pooled, ss)
    dh, dw, dws = torch.zeros_like(h), torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    with pytest.raises(_lib.HeroError):
        ops.qa_pool_bwd(h, fmap, mask, wv, None, a, None, d_pool, None, rows, 1, length, dh, dw,
                        dws)
    with pytest.raises(ValueError):           # bounds: before any launch
        ops.qa_pool_fwd(h, fmap, mask, wv, None, rows, 1, 513, a, None, pooled, None)


def test_model_matches_reference_fixture(tmp_path):
    vx = cpu.fixture()
    model = cpu.violin_model(tmp_path, vx).to(DEV)

    def batch():
        return {k: (v.to(DEV) if torch.is_tensor(v) else v)
                for k, v in cpu.qa.qa_batch(vx).items()}

    with torch.no_grad():
        logits = model(batch(), "violin", compute_loss=False).cpu().numpy()
        loss = model(batch())
    ref = vx["logits"]
    assert np.abs(logits - ref).max() <= 2e-2 * max(np.abs(ref).max(), 1.0)
    assert abs(float(loss) - float(vx["loss"])) < 2e-2
    model(batch()).backward()
    params = dict(model.named_parameters())
    for name in json.loads(str(vx["grad_params"])):
        rel = _rel(params[name].grad.cpu(), torch.from_numpy(vx["g." + name]))
        assert rel < 3e-2, (name, rel)


def _violin_model(seed=0):
    import tempfile
    from hero_b200.model import VideoModelConfig
    from hero_b200.violin import HeroForViolin
    from oracle import gen_golden as gg
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(gg.model_json(768, 3072, 12, 6, 3, 50272), f)
        path = f.name
    torch.manual_seed(seed)
    return HeroForViolin(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100), path


def _head_grads_nonzero(model):
    for mod in (model.violin_pool, model.violin_pred_head):
        for n, p in mod.named_parameters():
            assert p.grad is not None and float(p.grad.abs().sum()) > 0, n


def test_training_step_does_not_sync_with_the_host():
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    model, _ = _violin_model()
    model = model.to(DEV).train()
    b = attach_plan(synth.syn_violin(seed=5), kind="violin")
    b = synth.to_device(b, DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = model(b, "violin")
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(loss)
    _head_grads_nonzero(model)


def test_validate_violin_on_synthetic_batches():
    from hero_b200 import evalpass, synth
    from hero_b200.plan import attach_plan
    model, _ = _violin_model()
    model = model.to(DEV)
    loader = []
    for s, n in ((1, 5), (2, 1)):                       # the second batch has a single statement
        b = attach_plan(synth.syn_violin_batch(n_videos=n, n_statements=1, seed=s), kind="violin")
        b = synth.to_device(b, DEV)
        b["qids"] = [f"q{s}-{i}" for i in range(n)]
        loader.append(b)
    copies = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(t, *a, **k):
        copies.append(tuple(t.shape))
        return real_cpu(t, *a, **k)

    torch.cuda.set_sync_debug_mode("warn")
    try:
        torch.Tensor.cpu = counting_cpu
        val_log, results, logits = evalpass.validate_violin(model, loader, "val",
                                                            save_logits=True)
    finally:
        torch.Tensor.cpu = real_cpu
        torch.cuda.set_sync_debug_mode("default")
    assert len(copies) == 2
    assert set(results) == {"q1-0", "q1-1", "q1-2", "q1-3", "q1-4", "q2-0"}
    assert set(results.values()) <= {0, 1}
    assert set(val_log) == {"valid/val_loss", "valid/val_acc", "valid/val_ex_per_s"}
    assert np.isfinite(val_log["valid/val_loss"])
    for qid, (score,) in logits.items():
        assert results[qid] == int(1 / (1 + np.exp(-score)) > 0.5)


# Gradient of the pooling weight: its size depends on how far the frames of a row differ after the
# temporal transformer, which is little at a random initialisation. It is measured against the
# reference's own bf16-autocast run (SURVEY §8c yardstick: <= 1.5x its error) if it misses 3e-2;
# every other gradient <= 3e-2.
YARDSTICK_GRADS = ("violin_pool.weight",)


def test_real_dimensions_match_staged_reference():
    """6 + 3 layers, H 768, VIOLIN preset, eval mode: logits, loss, head and encoder gradients
    against the reference's HeroForViolin in fp32 on the same GPU (SURVEY §8c bounds), with the
    same reference under torch bf16 autocast as the yardstick."""
    VideoModelConfig, _ = qa_gpu._reference_module()
    from model.violin import HeroForViolin as RefViolin
    from hero_b200 import synth
    model, path = _violin_model(seed=3)
    ref = RefViolin(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(model.state_dict())
    model, ref = model.to(DEV).eval(), ref.to(DEV).eval()
    hb = synth.syn_violin(seed=9)
    outs = []
    for m, bf16 in ((model, False), (ref, False), (ref, True)):
        m.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
            logits = m(dict(synth.to_device(hb, DEV)), "violin", compute_loss=False)
        # the reference's loss expression, outside autocast (torch refuses binary_cross_entropy
        # under CUDA autocast)
        scores = torch.sigmoid(logits.float()).squeeze(-1)
        loss = F.binary_cross_entropy(scores, hb["targets"].to(DEV).squeeze(-1).float())
        loss.backward()
        outs.append((logits.detach().float(), loss.detach(),
                     {n: p.grad.detach().clone() for n, p in m.named_parameters()
                      if p.grad is not None}))
    (lo, so, go), (lr, sr, gr), (_, _, gb) = outs
    assert float((lo - lr).abs().max()) <= 2e-2 * max(float(lr.abs().max()), 1.0)
    assert abs(float(so) - float(sr)) < 2e-2
    # our model's own loss path gives the same loss
    with torch.no_grad():
        own = model(dict(synth.to_device(hb, DEV)), "violin")
    assert abs(float(own) - float(so)) < 1e-5
    heads = [n for n in gr if n.startswith(("violin_pool", "violin_pred_head"))]
    assert len(heads) == 7
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
        if n in YARDSTICK_GRADS and ours >= 3e-2:
            assert ours <= 1.5 * bf16, (n, ours, bf16)
        else:
            assert ours < 3e-2, (n, ours, bf16)


def test_prefetch_loader_stages_the_violin_plan():
    """PrefetchLoader builds (in-process fallback) or takes (collate-attached) both VIOLIN plans
    and uploads the QaPlan through the stager's buffers; the step then makes no host sync."""
    from hero_b200 import synth
    from hero_b200.loader import PrefetchLoader
    from hero_b200.plan import PLAN_KEY, QA_PLAN_KEY, attach_plan
    model, _ = _violin_model()
    model = model.to(DEV).train()
    host = [synth.syn_violin_batch(n_videos=2, seed=s) for s in (3, 4)]
    host[1] = attach_plan(host[1], kind="violin")
    n = 0
    for b in PrefetchLoader(host, device=DEV, depth=2):
        assert b[PLAN_KEY] is not None and b[QA_PLAN_KEY] is not None
        assert b[QA_PLAN_KEY].dev is not None and b[QA_PLAN_KEY].n_cand == 1
        model.zero_grad()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss = model(b, "violin")
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.isfinite(loss)
        _head_grads_nonzero(model)
        n += 1
    assert n == 2
