"""Host-side orchestration (plans + autograd chains + module plumbing) checked on CPU against
the reference-generated golden fixture, with `hero_b200.ops` monkeypatched to torch restatements
of the C-ABI contracts (tests/fake_ops.py). The CUDA kernels themselves are checked on the GPU
(tests/test_kernels_gpu.py, tests/test_encoder_gpu.py)."""
import json

import numpy as np
import torch

from tests import fake_ops
from tests import golden_util as gu


def _json(tmp_path, d):
    def cfg(n, v):
        c = {"attention_probs_dropout_prob": 0.1, "hidden_act": "gelu", "hidden_dropout_prob": 0.1,
             "hidden_size": d["hidden"], "initializer_range": 0.02,
             "intermediate_size": d["inter"], "max_position_embeddings": 514,
             "num_attention_heads": d["heads"], "num_hidden_layers": n, "type_vocab_size": 2}
        if v:
            c["vocab_size"] = d["vocab"]
        return c
    p = tmp_path / "m.json"
    p.write_text(json.dumps({"f_config": cfg(d["f_layers"], True),
                             "c_config": cfg(d["c_layers"], False)}))
    return str(p)


def _model(tmp_path, fx):
    from hero_b200.model import HierarchicalVlModel, VideoModelConfig
    d = gu.dims_of(fx)
    m = HierarchicalVlModel(VideoModelConfig(_json(tmp_path, d)), vfeat_dim=d["vfeat_dim"],
                            max_frm_seq_len=d["max_img_len"])
    missing, unexpected = m.load_state_dict(gu.weights_for(fx), strict=False)
    assert not unexpected
    return m.eval()


def _close(got, ref, mask, atol, what):
    got = got.detach().float().numpy()[mask]
    ref = ref[mask]
    err = np.abs(got - ref).max()
    assert err <= atol, f"{what}: max abs err {err}"


def test_forward_matches_reference_golden(tmp_path, monkeypatch):
    fake_ops.install(monkeypatch)
    fx = gu.load("hier_tiny.npz")
    model = _model(tmp_path, fx)
    vb, qb = gu.stored_batches(fx)
    with torch.no_grad():
        f_seq, pooled = model.f_encoder(vb, "repr")
        clip = model(vb, "repr")
        pre = model.forward_repr(vb, encode_clip=False)
        q = model.f_encoder(qb, "txt")[0]
    fm = vb["f_attn_masks"].bool().numpy()
    cm = vb["c_attn_masks"].bool().numpy()
    _close(f_seq, fx["f_seq_out"], fm, 6e-2, "f_encoder sequence output")
    _close(clip, fx["clip_out"], cm, 6e-2, "clip outputs")
    _close(pre, fx["pre_clip"], cm, 8e-2, "pre-temporal features")
    _close(q, fx["q_seq_out"], qb["attn_masks"].bool().numpy(), 6e-2, "query rows")
    assert float(clip.numpy()[~cm].max(initial=0.0)) == 0.0


def test_backward_matches_reference_golden(tmp_path, monkeypatch):
    fake_ops.install(monkeypatch)
    fx = gu.load("hier_tiny.npz")
    model = _model(tmp_path, fx)
    vb, qb = gu.stored_batches(fx)
    clip = model(vb, "repr")
    q = model.f_encoder(qb, "txt")[0]
    loss = (clip * torch.from_numpy(fx["loss_w1"])).sum() + (q * torch.from_numpy(fx["loss_w2"])).sum()
    assert abs(loss.item() - float(fx["loss"])) < 0.05 * max(1.0, abs(float(fx["loss"])))
    loss.backward()
    named = dict(model.named_parameters())
    for k, ref in fx.items():
        if not k.startswith("grad."):
            continue
        g = named[k[5:]].grad
        assert g is not None, k
        rel = np.linalg.norm(g.numpy() - ref) / max(np.linalg.norm(ref), 1e-12)
        assert rel < 4e-2, f"{k}: relative Frobenius error {rel}"


def test_generic_bert_encoder_and_temporal_apis(tmp_path, monkeypatch):
    fake_ops.install(monkeypatch)
    from oracle import hero_oracle as orc
    fx = gu.load("hier_tiny.npz")
    d = gu.dims_of(fx)
    model = _model(tmp_path, fx)
    P = gu.weights_for(fx)
    g = torch.Generator().manual_seed(4)
    h = torch.randn(3, 7, d["hidden"], generator=g)
    mask = torch.tensor([[1] * 7, [1, 1, 1, 0, 0, 0, 0], [0, 1, 1, 1, 1, 0, 0]])
    with torch.no_grad():
        out = model.c_encoder.encoder(h, mask)[0]
        tout = model.c_encoder(h, None, mask)
    ref = orc.bert_encoder(h, mask, P, "c_encoder.encoder.", d["c_layers"], d["heads"])
    _close(out, ref.numpy(), mask.bool().numpy(), 6e-2, "BertEncoder padded API")
    tref = orc.temporal_trm(P, "c_encoder.", h, mask, d["c_layers"], d["heads"])
    _close(tout, tref.numpy(), mask.bool().numpy(), 6e-2, "TemporalTrm.forward")


def test_plan_can_be_attached_at_collate_time(tmp_path, monkeypatch):
    """Plans attached at collate time give the outputs of the plans the forward builds itself,
    separately and in the fused joint pass."""
    fake_ops.install(monkeypatch)
    from hero_b200.plan import PLAN_KEY, attach_plan
    fx = gu.load("hier_tiny.npz")
    model = _model(tmp_path, fx)
    vb, qb = gu.stored_batches(fx)
    with torch.no_grad():
        a = model(vb, "repr")
        vb2 = attach_plan(dict(vb))
        assert PLAN_KEY in vb2
        b = model(vb2, "repr")
        qa = model.f_encoder(qb, "txt")[0]
        qb2 = attach_plan(dict(qb), kind="txt")
        qb_out = model.f_encoder(qb2, "txt")[0]
        ja, jqa = model.forward_repr_txt(dict(vb), dict(qb))
        jb, jqb = model.forward_repr_txt(vb2, qb2)
    assert torch.equal(a, b)
    assert torch.equal(qa, qb_out)
    assert torch.equal(ja, jb) and torch.equal(jqa, jqb)


def test_per_row_position_ids_give_the_shared_row_results(tmp_path, monkeypatch):
    """Position ids given per row (R, L) instead of once (1, L) read the same table rows: outputs
    and every gradient, the position table's included, are the same, plan attached or not."""
    fake_ops.install(monkeypatch)
    from hero_b200.plan import attach_plan
    fx = gu.load("hier_tiny.npz")
    vb, _ = gu.stored_batches(fx)
    w1 = torch.from_numpy(fx["loss_w1"])
    rows = dict(vb, f_sub_pos_ids=vb["f_sub_pos_ids"].expand_as(vb["f_sub_input_ids"]).clone())
    assert vb["f_sub_pos_ids"].shape[0] == 1 < rows["f_sub_pos_ids"].shape[0]

    def run(batch):
        model = _model(tmp_path, fx)
        clip = model(batch, "repr")
        (clip * w1).sum().backward()
        return clip.detach(), {k: p.grad for k, p in model.named_parameters()
                               if p.grad is not None}

    a, ga = run(vb)
    for batch in (rows, attach_plan(dict(rows))):
        b, gb = run(batch)
        assert torch.equal(a, b) and ga.keys() == gb.keys()
        for k in ga:
            assert torch.equal(ga[k], gb[k]), k


def test_in_place_gradient_sinks_match_autograd_accumulation(tmp_path, monkeypatch):
    """With FlatParams.ensure_flat_grads the backward accumulates straight into the flat gradient
    buffer (no zero-fill / add pass); the result must equal the plain autograd path, and a second
    backward must accumulate (+=) like autograd does."""
    fake_ops.install(monkeypatch)
    from hero_b200.params import flat_of
    fx = gu.load("hier_tiny.npz")
    vb, qb = gu.stored_batches(fx)
    w1, w2 = torch.from_numpy(fx["loss_w1"]), torch.from_numpy(fx["loss_w2"])

    def loss_of(model):
        clip = model(vb, "repr")
        q = model.f_encoder(qb, "txt")[0]
        return (clip * w1).sum() + (q * w2).sum()

    ref = _model(tmp_path, fx)
    loss_of(ref).backward()
    ref_grads = {k: p.grad.clone() for k, p in ref.named_parameters() if p.grad is not None}

    model = _model(tmp_path, fx)
    flat = flat_of(model, torch.device("cpu"))
    gflat = flat.ensure_flat_grads()
    loss_of(model).backward()
    for k, p in model.named_parameters():
        if k in ref_grads:
            assert torch.allclose(p.grad, ref_grads[k], rtol=1e-5, atol=1e-6), k
            assert p.grad.untyped_storage().data_ptr() == gflat.untyped_storage().data_ptr(), k
    loss_of(model).backward()
    for k, p in model.named_parameters():
        if k in ref_grads:
            assert torch.allclose(p.grad, 2 * ref_grads[k], rtol=1e-4, atol=1e-5), k


def test_fused_repr_txt_equals_separate_calls(tmp_path, monkeypatch):
    """forward_repr_txt (query rows ride along with the video rows) == the two reference calls,
    forward and backward."""
    fake_ops.install(monkeypatch)
    fx = gu.load("hier_tiny.npz")
    vb, qb = gu.stored_batches(fx)
    w1, w2 = torch.from_numpy(fx["loss_w1"]), torch.from_numpy(fx["loss_w2"])
    ref = _model(tmp_path, fx)
    clip_r = ref(vb, "repr")
    q_r = ref.f_encoder(qb, "txt")[0]
    ((clip_r * w1).sum() + (q_r * w2).sum()).backward()
    model = _model(tmp_path, fx)
    clip, q = model.forward_repr_txt(vb, qb)
    assert torch.allclose(clip, clip_r, atol=2e-2) and torch.allclose(q, q_r, atol=2e-2)
    cm = vb["c_attn_masks"].bool().numpy()
    _close(clip, fx["clip_out"], cm, 6e-2, "fused clip outputs")
    _close(q, fx["q_seq_out"], qb["attn_masks"].bool().numpy(), 6e-2, "fused query rows")
    ((clip * w1).sum() + (q * w2).sum()).backward()
    gr = dict(ref.named_parameters())
    for k, p in model.named_parameters():
        if gr[k].grad is None:
            continue
        rel = (p.grad - gr[k].grad).norm() / gr[k].grad.norm().clamp_min(1e-9)
        assert rel < 2e-2, (k, float(rel))


def test_bf16_mirror_follows_any_torch_optimizer_step(tmp_path, monkeypatch):
    """The kernels read a bf16 mirror of the fp32 masters. An optimizer that updates `p.data` in
    place (the reference's optim/adamw.py:94-104 does; `p._version` does not move) must still be
    seen by the next forward: FlatParams listens to every torch.optim.Optimizer.step()."""
    fake_ops.install(monkeypatch)
    from hero_b200.params import flat_of
    fx = gu.load("hier_tiny.npz")
    vb, _ = gu.stored_batches(fx)

    class DataSGD(torch.optim.Optimizer):      # updates through .data like the reference's AdamW
        def __init__(self, params):
            super().__init__(params, dict(lr=0.5))

        def step(self, closure=None):
            for group in self.param_groups:
                for p in group["params"]:
                    if p.grad is not None:
                        p.data.add_(p.grad.data, alpha=-group["lr"])

    model = _model(tmp_path, fx)
    flat = flat_of(model, torch.device("cpu"))
    opt = DataSGD(model.parameters())
    out0 = model(vb, "repr")
    out0.float().pow(2).mean().backward()
    assert not flat.dirty
    opt.step()
    assert flat.dirty                                  # marked by the global post-step hook
    out1 = model(vb, "repr")
    assert (out1 - out0).abs().max() > 1e-3            # the forward saw the new weights
    fresh = _model(tmp_path, fx)
    fresh.load_state_dict(model.state_dict())
    assert torch.equal(fresh(vb, "repr"), out1)


def test_fp16_checkpoint_round_trip_after_the_model_has_run(tmp_path, monkeypatch):
    """SURVEY.md 8f rank 4: checkpoints are written with the reference's conventions
    (utils/save.py:117-130: plain state_dict + a 'vocab_padded' flag, fp16 tensors on disk for the
    released weights) and must load into a model whose flat buffers already exist — the bf16
    working copy has to follow."""
    fake_ops.install(monkeypatch)
    from hero_b200.encoder import load_pretrained_weight
    fx = gu.load("hier_tiny.npz")
    vb, _ = gu.stored_batches(fx)
    src = _model(tmp_path, fx)
    ckpt = {k: v.half() for k, v in src.state_dict().items()}
    ckpt["vocab_padded"] = True
    path = tmp_path / "model_step_1.pt"
    torch.save(ckpt, str(path))

    dst = _model(tmp_path, fx)
    with torch.no_grad():
        for p in dst.parameters():
            p.mul_(0.5)                       # some other weights ...
    out_other = dst(vb, "repr")               # ... and the flat buffers + bf16 mirror exist
    load_pretrained_weight(dst, torch.load(str(path)))
    out_loaded = dst(vb, "repr")
    for (k, a), (_, b) in zip(dst.state_dict().items(), src.state_dict().items()):
        assert torch.equal(a, b.half().to(a.dtype)), k
    want = src(vb, "repr")
    m = vb["c_attn_masks"].bool()
    assert (out_loaded - out_other)[m].abs().max() > 1e-2
    assert (out_loaded - want)[m].abs().max() < 6e-2          # fp16-rounded weights, bf16 math


def test_batch_without_f_v_feats_reads_the_clip_frames(tmp_path, monkeypatch):
    """SURVEY.md 8f rank 2 (first step): `f_v_feats` is a row gather of `c_v_feats`; a batch that
    omits it (half the host->device bytes) must give exactly the same outputs and gradients, on
    the plain and on the fused query path. MFM keeps requiring it (c_v_feats is masked in place)."""
    import pytest
    fake_ops.install(monkeypatch)
    fx = gu.load("hier_tiny.npz")
    vb, qb = gu.stored_batches(fx)
    slim = {k: v for k, v in vb.items() if k != "f_v_feats"}
    w1 = torch.from_numpy(fx["loss_w1"])

    def run(batch, fused):
        model = _model(tmp_path, fx)
        if fused:
            clip, q = model.forward_repr_txt(batch, qb)
        else:
            clip, q = model(batch, "repr"), None
        (clip * w1).sum().backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        return clip.detach(), q, grads

    for fused in (False, True):
        a, qa, ga = run(vb, fused)
        b, qb_out, gb = run(slim, fused)
        assert torch.equal(a, b)
        if fused:
            assert torch.equal(qa, qb_out)
        assert ga.keys() == gb.keys()
        for k in ga:
            assert torch.equal(ga[k], gb[k]), k
    model = _model(tmp_path, fx)
    mb = dict(slim)
    mb["c_v_masks"] = torch.zeros_like(vb["c_attn_masks"], dtype=torch.bool)
    mb["c_v_masks"][:, 0] = True
    mb["feat_targets"] = vb["c_v_feats"][mb["c_v_masks"]]
    with pytest.raises(ValueError):
        model(mb, "mffr")


def test_fused_adamw_host_logic_groups_clipping_and_state_dict(monkeypatch):
    """FusedAdamW's host side on CPU (kernels replaced by their torch restatements): two launches
    over the decay / no-decay ranges == the reference rule per parameter (optim/adamw.py:80-104,
    grouping optim/misc.py:22), global-norm clipping folded into the update, the training loop's
    `for g in optimizer.param_groups: g['lr'] = ...` (train_vcmr.py:245-247), and a
    state_dict round trip (utils/save.py TrainingRestorer)."""
    from oracle import hero_oracle as orc
    fake_ops.install(monkeypatch)
    from hero_b200.optim import FusedAdamW
    from hero_b200.params import flat_of

    class Tiny(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.dense = torch.nn.Linear(96, 64)
            self.LayerNorm = torch.nn.LayerNorm(64)
            self.proj = torch.nn.Linear(64, 40)

    def make():
        torch.manual_seed(0)
        m = Tiny()
        flat = flat_of(m, torch.device("cpu"))
        return m, flat, FusedAdamW(flat, lr=1e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01)

    m, flat, opt = make()
    assert flat.no_decay_start < flat.total and len(opt.param_groups) == 2
    ref_p = {k: p.detach().clone() for k, p in m.named_parameters()}
    ref_m = {k: torch.zeros_like(v) for k, v in ref_p.items()}
    ref_v = {k: torch.zeros_like(v) for k, v in ref_p.items()}
    g = torch.Generator().manual_seed(1)
    lrs = [1e-3, 5e-4, 2e-3]
    saved = None
    for step in range(1, 4):
        opt.zero_grad()
        grads = {k: torch.randn(v.shape, generator=g) * 0.1 for k, v in ref_p.items()}
        for k, p in m.named_parameters():
            p.grad.copy_(grads[k])
        for grp in opt.param_groups:
            grp["lr"] = lrs[step - 1]
        total = torch.sqrt(sum((v.double() ** 2).sum() for v in grads.values())).item()
        assert abs(opt.clip_grad_norm_(1.0) - total) < 1e-3 * total
        scale = min(1.0, 1.0 / (total + 1e-6))
        opt.step()
        for k in ref_p:
            wd = 0.0 if ("bias" in k or "LayerNorm" in k) else 0.01
            ref_p[k], ref_m[k], ref_v[k] = orc.adamw_step(ref_p[k], grads[k] * scale, ref_m[k],
                                                          ref_v[k], step, lrs[step - 1], 0.9, 0.98,
                                                          1e-6, wd)
        for k, p in m.named_parameters():
            assert (p.detach() - ref_p[k]).abs().max() < 2e-6, (k, step)
        if step == 2:
            saved = ({k: v.clone() if torch.is_tensor(v) else v for k, v in
                      opt.state_dict().items()}, {k: v.clone() for k, v in m.state_dict().items()},
                     grads)
    assert not flat.dirty                              # the optimizer refreshed the bf16 mirror
    for k, p in m.named_parameters():
        assert torch.equal(flat.bf16(p), p.detach().to(torch.bfloat16)), k
    # resume from the step-2 snapshot and repeat step 3: same parameters
    m2, flat2, opt2 = make()
    m2.load_state_dict(saved[1])
    opt2.load_state_dict(saved[0])
    assert opt2.step_count == 2
    opt2.zero_grad()
    for k, p in m2.named_parameters():
        p.grad.copy_(grads[k])                         # `grads`: the step-3 gradients
    for grp in opt2.param_groups:
        grp["lr"] = lrs[2]
    opt2.clip_grad_norm_(1.0)
    opt2.step()
    for (k, a), (_, b) in zip(m2.named_parameters(), m.named_parameters()):
        assert (a.detach() - b.detach()).abs().max() < 1e-7, k


def test_model_saver_and_training_restorer_round_trip(tmp_path, monkeypatch):
    """SURVEY.md 8f rank 4: hero_b200.evalpass.ModelSaver / TrainingRestorer write the reference's
    file layout (utils/save.py:112-181): `model_step_<n>.pt` with a `vocab_padded` flag (fp16
    tensors on request), `train_state_<n>.pt`, rotating `restore.pt`; a fresh model + optimizer
    resume from them bit for bit (fp32) and keep training."""
    fake_ops.install(monkeypatch)
    from hero_b200.evalpass import ModelSaver, TrainingRestorer, load_checkpoint
    from hero_b200.optim import FusedAdamW
    from hero_b200.params import flat_of
    fx = gu.load("hier_tiny.npz")
    vb, _ = gu.stored_batches(fx)
    out_dir = tmp_path / "ckpt"
    out_dir.mkdir()

    def train_steps(model, opt, n):
        for _ in range(n):
            opt.zero_grad()
            model(vb, "repr").square().mean().backward()
            opt.step()

    src = _model(tmp_path, fx).train()
    for m in src.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    opt = FusedAdamW(flat_of(src, torch.device("cpu")), lr=1e-3)
    rest = TrainingRestorer(str(out_dir), src, opt, save_steps=2)
    train_steps(src, opt, 2)
    rest.step(); rest.step()                     # global_step 2 -> restore.pt written
    assert (out_dir / "restore.pt").exists()
    path = ModelSaver(str(out_dir), half=True).save(src, 2, opt)
    sd = torch.load(path)
    assert sd["vocab_padded"] is True
    assert all(v.dtype == torch.float16 for k, v in sd.items()
               if isinstance(v, torch.Tensor) and v.is_floating_point())
    assert set(k for k in sd if k != "vocab_padded") == set(src.state_dict())
    assert (out_dir / "train_state_2.pt").exists()

    # resume in a fresh model + optimizer: same weights, same moments, same next step
    dst = _model(tmp_path, fx).train()
    for m in dst.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    with torch.no_grad():
        for p in dst.parameters():
            p.add_(0.1)
    dst(vb, "repr")                              # flat buffers exist before the restore
    opt2 = FusedAdamW(flat_of(dst, torch.device("cpu")), lr=1e-3)
    rest2 = TrainingRestorer(str(out_dir), dst, opt2, save_steps=2)
    assert rest2.global_step == 2 and opt2.step_count == opt.step_count
    for (k, a), (_, b) in zip(dst.state_dict().items(), src.state_dict().items()):
        assert torch.equal(a, b), k
    assert torch.equal(opt2.exp_avg, opt.exp_avg) and torch.equal(opt2.exp_avg_sq, opt.exp_avg_sq)
    train_steps(src, opt, 1)
    train_steps(dst, opt2, 1)
    for (k, a), (_, b) in zip(dst.state_dict().items(), src.state_dict().items()):
        assert torch.allclose(a, b, atol=1e-6), k
    # fp16 model file loads into a model that has run
    load_checkpoint(dst, path)
    for (k, a), (_, b) in zip(dst.state_dict().items(), sd.items()):
        if isinstance(b, torch.Tensor):
            assert torch.equal(a, b.float().to(a.dtype)), k
