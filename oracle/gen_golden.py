"""Generates tests/golden/*.npz by running the UNMODIFIED reference modules on CPU.

Needs a checkout of the reference, given as HERO_REFERENCE=<path>; the GPU tests never run it.
The reference is imported, never copied: apex / horovod / lmdb ... are replaced by in-memory
stubs (SURVEY.md Appendix B), `FusedLayerNorm` by `torch.nn.LayerNorm` (same semantics and
parameter names). Fixtures hold outputs (and, for tiny configs, the weights and inputs); the
full-dimension fixtures regenerate weights/inputs from seeds via `oracle.hero_oracle.seeded_weights`
and `hero_b200.synth`, so the files stay small.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python oracle/gen_golden.py
"""
import itertools
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("HERO_REFERENCE", "")
sys.path.insert(0, ROOT)

from hero_b200 import synth  # noqa: E402
from oracle import hero_oracle as orc  # noqa: E402


def install_stubs():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    fln = mod("apex.normalization.fused_layer_norm", FusedLayerNorm=torch.nn.LayerNorm)
    mod("apex.normalization", fused_layer_norm=fln)
    mod("apex", normalization=sys.modules["apex.normalization"], amp=mod("apex.amp"))
    hvd = mod("horovod.torch", size=lambda: 1, rank=lambda: 0, local_rank=lambda: 0,
              local_size=lambda: 1, allgather=lambda t, name=None: t,
              allgather_async=lambda t, name=None: t, synchronize=lambda h: h)
    mod("horovod", torch=hvd)
    mod("lmdb")
    mod("lz4")
    mod("lz4.frame", compress=None, decompress=None)
    mod("msgpack_numpy", patch=lambda: None)
    mod("toolz")
    mod("toolz.sandbox", unzip=lambda seq: zip(*seq))
    mod("cytoolz", concat=itertools.chain.from_iterable)
    mod("tensorboardX", SummaryWriter=object)
    if not os.path.isfile(os.path.join(REF, "model", "model.py")):
        raise SystemExit("set HERO_REFERENCE to a checkout of linjieli222/HERO")
    sys.path.insert(0, REF)


def model_json(hidden, inter, heads, f_layers, c_layers, vocab, max_pos=514):
    def cfg(n_layers, with_vocab):
        c = {"attention_probs_dropout_prob": 0.1, "hidden_act": "gelu",
             "hidden_dropout_prob": 0.1, "hidden_size": hidden, "initializer_range": 0.02,
             "intermediate_size": inter, "max_position_embeddings": max_pos,
             "num_attention_heads": heads, "num_hidden_layers": n_layers, "type_vocab_size": 2}
        if with_vocab:
            c["vocab_size"] = vocab
        return c
    return {"f_config": cfg(f_layers, True), "c_config": cfg(c_layers, False)}


def build_reference_model(dims, weights):
    from model.model import HierarchicalVlModel, VideoModelConfig
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(model_json(dims["hidden"], dims["inter"], dims["heads"], dims["f_layers"],
                             dims["c_layers"], dims["vocab"]), f)
        path = f.name
    config = VideoModelConfig(path)
    os.unlink(path)
    model = HierarchicalVlModel(config, vfeat_dim=dims["vfeat_dim"],
                                max_frm_seq_len=dims["max_img_len"])
    missing, unexpected = model.load_state_dict(weights, strict=False)
    assert not unexpected, unexpected
    # everything on the encoder path must be covered by our seeded weights
    hot_missing = [k for k in missing if not (k.startswith(("feat_regress", "mask_embedding",
                                                              "fom_output", "pad",
                                                              "f_encoder.lm_head", "f_encoder.pad"))
                                              )]
    assert not hot_missing, hot_missing
    model.eval()
    return model


def ragged_batch(seed, dims, batch_size):
    vb, qb = synth.syn_tvr_ragged(batch_size=batch_size, seed=seed, vfeat_dim=dims["vfeat_dim"],
                                  vocab=dims["vocab"] - 7, t_range=(6, 14), s_range=(2, 5),
                                  l_range=(3, 9), q_range=(3, 8))
    return vb, qb


def check_collate_layout():
    """The synthetic generator must reproduce the reference's own video_collate layout."""
    from data.data import video_collate
    gen = torch.Generator().manual_seed(5)
    clips = []
    specs = [(9, [[0, 1, 2], [], [5, 6]], [4, 6, 3]), (5, [[1], [2, 3, 4]], [7, 2])]
    for T, frames, lens in specs:
        clips.append(synth.make_clip(gen, T, frames, lens, vfeat_dim=16, vocab=50))
    mine = synth.video_batch(clips)
    items = []
    for c in clips:
        T = c["feats"].shape[0]
        ids, feats, masks = [], [], []
        for sub, (_, fr) in zip(c["subs"], c["sub2frames"]):
            fr = [f for f in fr if f in range(T)]
            if fr:
                feats.append(torch.index_select(c["feats"], 0, torch.tensor(fr)))
                masks.append(torch.tensor([1] * (len(sub) + len(fr))))
            else:
                feats.append(torch.zeros(1, c["feats"].shape[1]))
                masks.append(torch.tensor([0] + [1] * len(sub)))
            ids.append(sub)
        items.append((ids, feats, masks, c["feats"], torch.tensor([1] * T), len(c["subs"]),
                      c["sub2frames"]))
    ref = video_collate(items)
    for k in ("f_sub_input_ids", "f_sub_pos_ids", "f_v_feats", "f_v_pos_ids", "f_attn_masks",
              "f_gather_index", "c_v_feats", "c_attn_masks"):
        assert torch.equal(ref[k], mine[k]), k
    assert ref["num_subs"] == mine["num_subs"]
    assert ref["sub_idx2frame_idx"] == mine["sub_idx2frame_idx"]
    print("synthetic collate layout == reference video_collate")


def heads_fixture(model, dims, vb, out_dir):
    """Pretraining heads of the reference on the tiny model (SURVEY.md 8f rank 3): MFM regression
    and NCE (model/model.py:239-289), FOM (:306-336) and MLM (model/encoder.py:355-374). The head
    parameters are not part of the seeded encoder weights: they are drawn here and stored."""
    gen = torch.Generator().manual_seed(77)
    head = {}
    for k, p in model.named_parameters():
        if k.startswith(("feat_regress", "fom_output", "mask_embedding", "f_encoder.lm_head.dense",
                         "f_encoder.lm_head.LayerNorm", "f_encoder.lm_head.bias")):
            with torch.no_grad():
                if p.dim() > 1:
                    p.copy_(torch.randn(p.shape, generator=gen) * 0.05)
                elif "LayerNorm.weight" in k:
                    p.copy_(1.0 + torch.randn(p.shape, generator=gen) * 0.05)
                else:
                    p.copy_(torch.randn(p.shape, generator=gen) * 0.05)
            head["head." + k] = p.detach().numpy().copy()
    with torch.no_grad():
        model.mask_embedding.weight[0].zero_()          # padding row (init_type_embedding)
    head["head.mask_embedding.weight"] = model.mask_embedding.weight.detach().numpy().copy()
    B, T = vb["c_attn_masks"].shape
    valid = vb["c_attn_masks"].bool()
    # ---- MFM: mask ~1/3 of the valid frames (at least one masked and one unmasked per clip)
    c_v_masks = (torch.rand(B, T, generator=gen) < 0.34) & valid
    for b in range(B):
        n = int(valid[b].sum())
        c_v_masks[b, 0], c_v_masks[b, n - 1] = True, False
    feat_targets = vb["c_v_feats"][c_v_masks].clone()

    def mfm_batch():
        b = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in vb.items()}
        b["c_v_masks"], b["feat_targets"] = c_v_masks.clone(), feat_targets.clone()
        return b

    with torch.no_grad():
        mffr_pred = model(mfm_batch(), "mffr", compute_loss=False)
        mffr_loss = model(mfm_batch(), "mffr", compute_loss=True)
        nce_loss = model(mfm_batch(), "mfm-nce", compute_loss=True)
    # ---- FOM: permute the valid frames of every clip; a third of the targets ignored (-1)
    orders = torch.arange(T).repeat(B, 1)
    targets = torch.full((B, T), -1, dtype=torch.long)
    for b in range(B):
        n = int(valid[b].sum())
        perm = torch.randperm(n, generator=gen)
        orders[b, :n] = perm
        keep = torch.rand(n, generator=gen) < 0.67
        targets[b, :n] = torch.where(keep, perm, torch.full((n,), -1))
    fb = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in vb.items()}
    fb["shuffled_orders"], fb["targets"] = orders, targets
    with torch.no_grad():
        fom_logits = model(fb, "fom", compute_loss=False)
        fom_loss = model(fb, "fom", compute_loss=True)
    # ---- MLM on the cross-modal rows: mask one or two text positions per row
    am = vb["f_attn_masks"]
    rows, L = am.shape
    max_vl = vb["f_v_feats"].shape[1]
    gi = vb["f_gather_index"]
    txt_mask_tgt = torch.zeros(rows, L, dtype=torch.bool)
    for r in range(rows):
        n = int(am[r].sum())
        # packed row = [frames, text, filler]: text slots are those gathered from >= max_vl
        text_pos = [j for j in range(L) if am[r, j] and int(gi[r, j]) >= max_vl]
        pick = torch.randperm(len(text_pos), generator=gen)[:2 if n > 6 else 1]
        for i in pick.tolist():
            txt_mask_tgt[r, text_pos[i]] = True
    n_masked = int(txt_mask_tgt.sum())
    txt_labels = torch.randint(5, dims["vocab"] - 8, (n_masked,), generator=gen)
    mb = {"input_ids": vb["f_sub_input_ids"], "position_ids": vb["f_sub_pos_ids"],
          "v_feat": vb["f_v_feats"], "f_pos_ids": vb["f_v_pos_ids"], "attn_masks": am,
          "gather_index": gi, "txt_mask_tgt": txt_mask_tgt, "txt_labels": txt_labels}
    with torch.no_grad():
        mlm_scores = model.f_encoder(mb, "mlm", compute_loss=False)
        mlm_loss = model.f_encoder(mb, "mlm", compute_loss=True)
    np.savez_compressed(
        os.path.join(out_dir, "heads_tiny.npz"), **head,
        c_v_masks=c_v_masks.numpy(), feat_targets=feat_targets.numpy(),
        mffr_pred=mffr_pred.numpy(), mffr_loss=mffr_loss.numpy(), nce_loss=nce_loss.numpy(),
        shuffled_orders=orders.numpy(), fom_targets=targets.numpy(),
        fom_logits=fom_logits.numpy(), fom_loss=np.float64(fom_loss.item()),
        txt_mask_tgt=txt_mask_tgt.numpy(), txt_labels=txt_labels.numpy(),
        mlm_scores=mlm_scores.numpy(), mlm_loss=mlm_loss.numpy())
    print("heads_tiny.npz: mffr", tuple(mffr_pred.shape), "nce", float(nce_loss.mean()),
          "fom", float(fom_loss), "mlm", tuple(mlm_scores.shape))


def vsm_fixture(dims, weights, vb, out_dir):
    """VSM / VCMR head of the reference (model/pretrain.py, model/vcmr.py; SURVEY.md 8f rank 1) on
    the tiny encoder: two queries per clip, eval mode (no dropout, 'sum' reductions), span logits,
    video-level scores and the three losses, plus the hard-negative weighting variant."""
    from model.vcmr import HeroForVcmr
    from model.model import VideoModelConfig
    cfgd = model_json(dims["hidden"], dims["inter"], dims["heads"], dims["f_layers"],
                      dims["c_layers"], dims["vocab"])
    cfgd["q_config"] = dict(cfgd["c_config"], num_hidden_layers=1)
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(cfgd, f)
        path = f.name
    config = VideoModelConfig(path)
    os.unlink(path)
    model = HeroForVcmr(config, vfeat_dim=dims["vfeat_dim"], max_frm_seq_len=dims["max_img_len"],
                        lw_neg_ctx=8, lw_neg_q=8, lw_st_ed=0.01, margin=0.1)
    missing, unexpected = model.load_state_dict(
        {"v_encoder." + k: v for k, v in weights.items()}, strict=False)
    assert not unexpected, unexpected
    gen = torch.Generator().manual_seed(91)
    head = {}
    for k, p in model.named_parameters():
        if k.startswith(("video_query_linear", "video_st_predictor", "video_ed_predictor",
                         "q_feat_attn")):
            with torch.no_grad():
                if "LayerNorm.weight" in k:
                    p.copy_(1.0 + torch.randn(p.shape, generator=gen) * 0.05)
                else:
                    p.copy_(torch.randn(p.shape, generator=gen) * (0.3 if "predictor" in k else 0.05))
            head["head." + k] = p.detach().numpy().copy()
    model.eval()
    B, T = vb["c_attn_masks"].shape
    k = 2                                           # queries per clip, grouped by clip
    Lq = 7
    q_ids = torch.randint(5, dims["vocab"] - 8, (B * k, Lq), generator=gen)
    q_len = torch.randint(3, Lq + 1, (B * k,), generator=gen)
    q_mask = (torch.arange(Lq)[None, :] < q_len[:, None]).long()
    q_ids = q_ids * q_mask + (1 - q_mask)           # padding id 1
    q_pos = torch.arange(Lq).unsqueeze(0)
    n_frames = vb["c_attn_masks"].sum(1)
    st = torch.stack([torch.randint(0, int(n_frames[i // k]), (1,), generator=gen)[0]
                      for i in range(B * k)])
    ed = torch.minimum(st + 2, n_frames.repeat_interleave(k) - 1)
    targets = torch.stack([st, ed], 1)
    targets[1] = -1                                  # one ignored query
    q_vidx = torch.arange(B).repeat_interleave(k)

    def batch():
        b = {kk: (v.clone() if torch.is_tensor(v) else v) for kk, v in vb.items()}
        b.update(query_input_ids=q_ids, query_pos_ids=q_pos, query_attn_masks=q_mask,
                 targets=targets, q_vidx=q_vidx)
        return b

    with torch.no_grad():
        scores, st_prob, ed_prob = model(batch(), "tvr", compute_loss=False)
        l_st_ed, l_ctx, l_q = model(batch(), "tvr", compute_loss=True)
        model.set_hard_negative(True, 2, 10)
        _, h_ctx, h_q = model(batch(), "tvr", compute_loss=True)
        model.set_hard_negative(False, 20, 10)
        model.ranking_loss_type = "lse"
        _, e_ctx, e_q = model(batch(), "tvr", compute_loss=True)
        model.ranking_loss_type = "hinge"
    # second batch: clips of EQUAL length (no padded frames), one query per clip -> the
    # non-cross span path and a span loss that does not depend on what the encoder leaves at
    # padded positions (hero_b200 zero-fills them, the reference does not)
    vbd, qbd = synth.syn_tvr_ragged(batch_size=3, seed=33, vfeat_dim=dims["vfeat_dim"],
                                    vocab=dims["vocab"] - 7, t_range=(9, 9), s_range=(2, 4),
                                    l_range=(3, 8), q_range=(3, 7))
    assert bool(vbd["c_attn_masks"].all())
    d_targets = torch.tensor([[1, 3], [0, 8], [4, 4]])

    def dense():
        b = {kk: (v.clone() if torch.is_tensor(v) else v) for kk, v in vbd.items()}
        b.update(query_input_ids=qbd["input_ids"], query_pos_ids=qbd["pos_ids"],
                 query_attn_masks=qbd["attn_masks"], targets=d_targets)
        return b

    with torch.no_grad():
        d_scores, d_st, d_ed = model(dense(), "tvr", compute_loss=False)
        d_l_st_ed, d_l_ctx, d_l_q = model(dense(), "tvr", compute_loss=True)
    dense_np = {"vbd." + k: v for k, v in np_batch(vbd).items()}
    dense_np.update({"qbd." + k: v for k, v in np_batch(qbd).items()})
    np.savez_compressed(
        os.path.join(out_dir, "vsm_tiny.npz"), **head, q_config=json.dumps(cfgd["q_config"]),
        state_dict_shapes=json.dumps({kk: list(v.shape) for kk, v in model.state_dict().items()}),
        query_input_ids=q_ids.numpy(), query_pos_ids=q_pos.numpy(),
        query_attn_masks=q_mask.numpy(), targets=targets.numpy(), q_vidx=q_vidx.numpy(),
        scores=scores.numpy(), st_prob=st_prob.numpy(), ed_prob=ed_prob.numpy(),
        loss_st_ed=l_st_ed.numpy(), loss_neg_ctx=l_ctx.numpy(), loss_neg_q=l_q.numpy(),
        hard_neg_ctx=h_ctx.numpy(), hard_neg_q=h_q.numpy(), lse_neg_ctx=e_ctx.numpy(),
        lse_neg_q=e_q.numpy(), **dense_np, d_num_subs=json.dumps(vbd["num_subs"]),
        d_sub_idx2frame_idx=json.dumps(vbd["sub_idx2frame_idx"]), d_targets=d_targets.numpy(),
        d_scores=d_scores.numpy(), d_st=d_st.numpy(), d_ed=d_ed.numpy(),
        d_loss_st_ed=d_l_st_ed.numpy(), d_loss_neg_ctx=d_l_ctx.numpy(),
        d_loss_neg_q=d_l_q.numpy())
    print("vsm_tiny.npz: scores", tuple(scores.shape), "st", tuple(st_prob.shape),
          "loss_st_ed", float(l_st_ed.sum()), "ctx", l_ctx.tolist())


def np_batch(b):
    return {k: v.numpy() for k, v in b.items() if torch.is_tensor(v)}


def main():
    install_stubs()
    torch.manual_seed(0)
    torch.set_grad_enabled(True)
    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    check_collate_layout()

    # ---- G1/G2: tiny dims, weights + inputs + outputs + a few gradients stored -----------------
    tiny = dict(hidden=128, inter=256, heads=2, f_layers=2, c_layers=2, vocab=120, vfeat_dim=64,
                max_img_len=20)
    shapes = orc.param_shapes(tiny["hidden"], tiny["inter"], tiny["f_layers"], tiny["c_layers"],
                              tiny["vocab"], 514, 2, tiny["vfeat_dim"], tiny["max_img_len"])
    W = orc.seeded_weights(shapes, seed=11, std=0.05)
    model = build_reference_model(tiny, W)
    vb, qb = ragged_batch(21, tiny, batch_size=3)
    f_out = model.f_encoder(vb, "repr")
    clip = model(vb, "repr")
    pre_clip = model.forward_repr(vb, encode_clip=False)
    q_out = model.f_encoder(qb, "txt")
    # gradient pin: scalar loss = sum(clip * w1) + sum(q_seq * w2) on valid positions
    gen = torch.Generator().manual_seed(3)
    w1 = torch.randn(clip.shape, generator=gen) * vb["c_attn_masks"].unsqueeze(-1)
    w2 = torch.randn(q_out[0].shape, generator=gen) * qb["attn_masks"].unsqueeze(-1)
    model.zero_grad()
    loss = (clip * w1).sum() + (q_out[0] * w2).sum()
    loss.backward()
    grad_keys = ["f_encoder.encoder.layer.0.attention.self.query.weight",
                 "f_encoder.encoder.layer.1.output.dense.bias",
                 "f_encoder.embeddings.word_embeddings.weight",
                 "f_encoder.embeddings.position_embeddings.weight",
                 "f_encoder.embeddings.token_type_embeddings.weight",
                 "f_encoder.img_embeddings.img_linear.weight",
                 "f_encoder.img_embeddings.img_LayerNorm.weight",
                 "f_encoder.img_embeddings.position_embeddings.weight",
                 "f_encoder.img_embeddings.LayerNorm.bias",
                 "frame_transform.LayerNorm.weight", "frame_transform.net.1.weight",
                 "c_encoder.embeddings.position_embeddings.weight",
                 "c_encoder.embeddings.LayerNorm.weight",
                 "c_encoder.encoder.layer.1.intermediate.dense.weight",
                 "c_encoder.encoder.layer.0.attention.output.LayerNorm.weight"]
    named = dict(model.named_parameters())
    grads = {"grad." + k: named[k].grad.numpy() for k in grad_keys}
    np.savez_compressed(
        os.path.join(out_dir, "hier_tiny.npz"),
        dims=json.dumps(tiny), seed_weights=11, weight_std=0.05,
        num_subs=json.dumps(vb["num_subs"]), sub_idx2frame_idx=json.dumps(vb["sub_idx2frame_idx"]),
        **{"vb." + k: v for k, v in np_batch(vb).items()},
        **{"qb." + k: v for k, v in np_batch(qb).items()},
        f_seq_out=f_out[0].detach().numpy(), f_pooled=f_out[1].detach().numpy(),
        clip_out=clip.detach().numpy(), pre_clip=pre_clip.detach().numpy(),
        q_seq_out=q_out[0].detach().numpy(), loss_w1=w1.numpy(), loss_w2=w2.numpy(),
        loss=np.float64(loss.item()), **grads)
    print("hier_tiny.npz: loss", loss.item())
    heads_fixture(model, tiny, vb, out_dir)
    vsm_fixture(tiny, W, vb, out_dir)

    # ---- G3: config 1 (SYN-XM-1), real dims, 1-layer CrossModalTrm -----------------------------
    full1 = dict(hidden=768, inter=3072, heads=12, f_layers=1, c_layers=1, vocab=50272,
                 vfeat_dim=4352, max_img_len=100)
    shapes = orc.param_shapes(f_layers=1, c_layers=1)
    W = orc.seeded_weights(shapes, seed=0)
    model = build_reference_model(full1, W)
    xb = synth.syn_xm_1(seed=0)
    with torch.no_grad():
        seq, pooled = model.f_encoder(xb, "repr")
    np.savez_compressed(os.path.join(out_dir, "xm1_config1.npz"), dims=json.dumps(full1),
                        seed_weights=0, seed_batch=0, seq_out=seq.numpy(), pooled=pooled.numpy())
    print("xm1_config1.npz", tuple(seq.shape))
    del model

    # ---- G4: full-depth encoder (hero_finetune dims), small ragged batch -----------------------
    full = dict(hidden=768, inter=3072, heads=12, f_layers=6, c_layers=3, vocab=50272,
                vfeat_dim=4352, max_img_len=100)
    shapes = orc.param_shapes()
    W = orc.seeded_weights(shapes, seed=1)
    model = build_reference_model(full, W)
    vb, qb = synth.syn_tvr_ragged(batch_size=2, seed=77, t_range=(10, 16), s_range=(3, 5),
                                  l_range=(4, 12), q_range=(5, 9))
    with open(os.path.join(out_dir, "state_dict_keys.json"), "w") as f:
        json.dump({k: list(v.shape) for k, v in model.state_dict().items()}, f, indent=0,
                  sort_keys=True)
    with torch.no_grad():
        clip = model(vb, "repr")
        q_seq = model.f_encoder(qb, "txt")[0]
    np.savez_compressed(os.path.join(out_dir, "hier_full_small.npz"), dims=json.dumps(full),
                        seed_weights=1, seed_batch=77, clip_out=clip.numpy(), q_seq_out=q_seq.numpy(),
                        c_attn_masks=vb["c_attn_masks"].numpy())
    print("hier_full_small.npz", tuple(clip.shape), tuple(q_seq.shape))

    # ---- G5: reference AdamW, three steps on a small tensor -------------------------------------
    from optim.adamw import AdamW
    gen = torch.Generator().manual_seed(9)
    p0 = torch.randn(257, generator=gen) * 0.1
    gs = [torch.randn(257, generator=gen) * 0.01 for _ in range(3)]
    p = torch.nn.Parameter(p0.clone())
    opt = AdamW([{"params": [p], "weight_decay": 0.01}], lr=1e-4, betas=(0.9, 0.98))
    traj = []
    for g in gs:
        p.grad = g.clone()
        opt.step()
        traj.append(p.detach().clone().numpy())
    np.savez_compressed(os.path.join(out_dir, "adamw.npz"), p0=p0.numpy(),
                        grads=np.stack([g.numpy() for g in gs]), traj=np.stack(traj),
                        lr=1e-4, beta1=0.9, beta2=0.98, eps=1e-6, weight_decay=0.01)
    print("adamw.npz")


if __name__ == "__main__":
    main()
