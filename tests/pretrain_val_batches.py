"""TEST INFRASTRUCTURE: the seeded pretraining validation batches of tests/golden/pretrain_val_tiny.npz
(two per task, from hero_b200.synth on ragged tiny clips), shared by tools/gen_pretrain_val_golden.py
and the tests, so the fixture stores results and seeds rather than inputs. Tiny configuration of
the other fixtures: H 128, vocabulary 120, 64-d frame features. The RoBERTa <mask> id of the
synthetic MLM batches lies outside the tiny vocabulary and is replaced by its last id."""
import torch

from hero_b200 import synth

H, INTER, HEADS, F_LAYERS, C_LAYERS, Q_LAYERS, VOCAB = 128, 256, 2, 2, 2, 1, 120
VFEAT, MAX_FRM = 64, 20
MASK_TINY = VOCAB - 1
WEIGHT_SEED, WEIGHT_STD = 13, 0.1
LOSS_WEIGHTS = dict(lw_neg_ctx=8, lw_neg_q=8, lw_st_ed=0.01)
TASKS = ("mlm", "mffr", "mfm-nce", "fom", "vsm")
SEEDS = (31, 32)


def model_json():
    from oracle import gen_golden as gg
    j = gg.model_json(H, INTER, HEADS, F_LAYERS, C_LAYERS, VOCAB)
    j["q_config"] = dict(j["c_config"], num_hidden_layers=Q_LAYERS)
    return j


def _video(seed, t_range=(6, 14)):
    return synth.syn_tvr_ragged(batch_size=3, seed=seed, vfeat_dim=VFEAT, vocab=VOCAB - 8,
                                t_range=t_range, s_range=(2, 5), l_range=(3, 9), q_range=(3, 8))


def batch(task, i):
    """Host batch i (0 or 1) of `task`, in the reference's collate layout for that task."""
    seed = SEEDS[i]
    # VSM: clips of equal length, so the span logits do not depend on what the encoder leaves at
    # padded frames (hero_b200 zero-fills them, the reference does not: hero_b200/pretrain.py)
    vb, qb = _video(seed, (10, 10) if task == "vsm" else (6, 14))
    if task == "mlm":
        b = synth.syn_mlm_batch(vb, seed=seed, mask_prob=0.3, vocab=VOCAB - 8)
        b["input_ids"] = b["input_ids"].masked_fill(b["input_ids"] == synth.MASK_ID, MASK_TINY)
        return b
    if task in ("mffr", "mfm-nce"):
        return synth.syn_mfm_batch(vb, seed=seed, mask_prob=0.3)
    if task == "fom":
        b = synth.syn_fom_batch(vb, seed=seed, reorder_p=0.5)
        b["vids"] = [f"v{seed}_{k}" for k in range(vb["c_attn_masks"].shape[0])]
        return b
    if task == "vsm":
        b = synth.syn_vsm_batch(vb, qb, seed=seed)
        b["q_vidx"] = torch.arange(vb["c_attn_masks"].shape[0])
        return b
    raise ValueError(task)


class Opts:
    lw_st_ed = LOSS_WEIGHTS["lw_st_ed"]
    lw_neg_ctx = LOSS_WEIGHTS["lw_neg_ctx"]
    lw_neg_q = LOSS_WEIGHTS["lw_neg_q"]


# ---- real dimensions (6 + 3 layers, H 768, vocabulary 50 272, 4352-d features) on
# SYN-HT100M-dense clips: the accuracy test of the fused MLM / MFM-NCE paths and the speed probe
REAL_VFEAT, REAL_VOCAB = 4352, 50272


def real_model(device, seed=0):
    """HeroForPretraining at real dimensions with its own initialisation (seeded), eval mode."""
    import json
    import os
    import tempfile
    from oracle import gen_golden as gg
    from hero_b200.model import VideoModelConfig
    from hero_b200.pretrain import HeroForPretraining
    j = gg.model_json(768, 3072, 12, 6, 3, REAL_VOCAB)
    j["q_config"] = dict(j["c_config"], num_hidden_layers=1)
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(j, f)
        path = f.name
    torch.manual_seed(seed)
    model = HeroForPretraining(VideoModelConfig(path), vfeat_dim=REAL_VFEAT, max_frm_seq_len=100,
                               **LOSS_WEIGHTS)
    os.unlink(path)
    return model.to(device).eval()


def real_batch(task, i, batch_size=8):
    """Host batch i of `task` on SYN-HT100M-dense clips (30 frames, 6 subtitles of 5 frames + 20
    tokens per clip)."""
    seed = 100 + i
    vb, qb = synth.syn_ht100m_dense(batch_size=batch_size, seed=seed, vfeat_dim=REAL_VFEAT)
    if task == "mlm":
        return synth.syn_mlm_batch(vb, seed=seed)
    if task in ("mffr", "mfm-nce"):
        return synth.syn_mfm_batch(vb, seed=seed)
    if task == "fom":
        b = synth.syn_fom_batch(vb, seed=seed)
        b["vids"] = [f"v{seed}_{k}" for k in range(batch_size)]
        return b
    if task == "vsm":
        b = synth.syn_vsm_batch(vb, qb, seed=seed)
        b["q_vidx"] = torch.arange(batch_size)
        return b
    raise ValueError(task)


@torch.no_grad()
def torch_logit_metrics(model, task, batches, autocast=False):
    """(summed cross entropy, top-1 hits, rows, per-row top-1 / top-2 gap) of MLM or MFM-NCE from
    the model's own torch logits (`compute_loss=False`: fp32 head.decoder / mfm_nce matmuls), the
    whole call under bf16 autocast when `autocast`."""
    import torch.nn.functional as F
    loss, hits, n, gaps = 0.0, 0, 0, []
    for b in batches:
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            if task == "mlm":
                logits = model(dict(b), task="mlm", compute_loss=False)
                labels = b["txt_labels"].to(logits.device)
            else:
                feats, neg = model(dict(b), task="mfm-nce", compute_loss=False)
                logits = model.v_encoder.mfm_nce(feats, b["feat_targets"], neg, compute_loss=False)
                labels = torch.arange(logits.shape[0], device=logits.device)
        logits = logits.float()
        loss += float(F.cross_entropy(logits, labels, reduction="sum"))
        hits += int((logits.max(dim=-1)[1] == labels).sum())
        n += int(labels.shape[0])
        top2 = logits.topk(2, dim=-1).values
        gaps.append(top2[:, 0] - top2[:, 1])
    return loss, hits, n, torch.cat(gaps)
