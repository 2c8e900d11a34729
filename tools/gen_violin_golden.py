"""Writes tests/golden/violin_tiny.npz: the reference's HeroForViolin (model/violin.py) on the tiny
configuration of tests/golden/videoqa_tiny.npz and a ragged VIOLIN training batch.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_violin_golden.py

It first checks that `hero_b200.synth.syn_violin_batch` equals the reference's own
`violin_collate` (data/violin.py:118-141) applied to the same dataset items, built the way
ViolinDataset.__getitem__ builds them (data/violin.py:63-115).

Configuration: H = 128, 2 heads, 2 cross-modal + 2 temporal layers, vocabulary 120, 64-d frame
features. Weights are `oracle.hero_oracle.seeded_weights` over the reference's state_dict shapes
(seed WEIGHT_SEED; rebuilt by the tests from the stored shape list), model in eval mode; the
batch is 3 videos x 2 statements (a true / false pair each), ragged clips, with joint
[frames | statement] rows both over and under 128 tokens. Stored: the batch, the reference's
state_dict key / shape list, the logits and the loss, and the gradients of the loss for the
parameters listed in GRAD_PARAMS: every head parameter (with a sigmoid loss none of them has a
zero gradient) plus the encoder parameters of the video QA fixture.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import synth  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import hero_oracle as orc  # noqa: E402

H, INTER, HEADS, F_LAYERS, C_LAYERS, VOCAB = 128, 256, 2, 2, 2, 120
VFEAT, MAX_FRM = 64, 120
WEIGHT_SEED, WEIGHT_STD = 7, 0.1
GRAD_PARAMS = (
    "violin_pool.weight",
    "violin_pred_head.linear_1.weight", "violin_pred_head.linear_1.bias",
    "violin_pred_head.LayerNorm.weight", "violin_pred_head.LayerNorm.bias",
    "violin_pred_head.linear_2.weight", "violin_pred_head.linear_2.bias",
    "v_encoder.c_encoder.encoder.layer.0.attention.self.query.weight",
    "v_encoder.c_encoder.encoder.layer.0.attention.self.key.weight",
    "v_encoder.c_encoder.encoder.layer.0.attention.self.value.weight",
    "v_encoder.c_encoder.embeddings.position_embeddings.weight",
    "v_encoder.f_encoder.embeddings.word_embeddings.weight",
    "v_encoder.f_encoder.encoder.layer.0.output.dense.weight",
)
BATCH_ARGS = dict(n_videos=3, n_statements=2, seed=13, t_range=(6, 110), s_range=(2, 5),
                  l_range=(3, 10), q_range=(8, 40), vfeat_dim=VFEAT, vocab=VOCAB)


def batch():
    return synth.syn_violin_batch(**BATCH_ARGS)


def reference_item(item):
    """ViolinDataset.__getitem__'s output for one synthetic item: per statement the video inputs
    with the statement appended to every subtitle (ids and attention masks)."""
    c = item["clip"]
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
    video_q, q_ids, q_masks, vids, targets = [], [], [], [], []
    for st, t in zip(item["statements"], item["targets"]):
        q_mask = torch.tensor([1] * len(st))
        video_q.append(([torch.cat((i, st)) for i in ids], feats,
                        [torch.cat((m, q_mask)) for m in masks], c["feats"],
                        torch.tensor([1] * T), len(c["subs"]), c["sub2frames"]))
        q_ids.append(st)
        q_masks.append(q_mask)
        vids.append("v")
        targets.append(torch.LongTensor([t]))
    return video_q, q_ids, q_masks, vids, targets


def check_violin_collate():
    from data.violin import violin_collate
    for args in (BATCH_ARGS, dict(BATCH_ARGS, n_statements=1, seed=4)):
        ref = violin_collate([reference_item(it) for it in synth.syn_violin_items(**args)])
        mine = synth.syn_violin_batch(**args)
        for k in ("f_sub_input_ids", "f_sub_pos_ids", "f_v_feats", "f_v_pos_ids", "f_attn_masks",
                  "f_gather_index", "c_v_feats", "c_attn_masks", "targets", "q_input_ids",
                  "q_pos_ids", "q_attn_masks"):
            assert torch.equal(ref[k], mine[k]), k
        assert ref["num_subs"] == mine["num_subs"]
        assert ref["sub_idx2frame_idx"] == mine["sub_idx2frame_idx"]
    print("syn_violin_batch == reference violin_collate")


def main():
    gg.install_stubs()
    check_violin_collate()
    from model.model import VideoModelConfig
    from model.violin import HeroForViolin
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(gg.model_json(H, INTER, HEADS, F_LAYERS, C_LAYERS, VOCAB), f)
        path = f.name
    config = VideoModelConfig(path)
    os.unlink(path)
    model = HeroForViolin(config, vfeat_dim=VFEAT, max_frm_seq_len=MAX_FRM).eval()
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(orc.seeded_weights(shapes, seed=WEIGHT_SEED, std=WEIGHT_STD))
    b = batch()
    lens = b["c_attn_masks"].sum(1) + b["q_attn_masks"].sum(1)
    assert int(lens.max()) > 128 and int(lens.min()) <= 128, lens
    out = {"config": json.dumps(dict(hidden=H, inter=INTER, heads=HEADS, f_layers=F_LAYERS,
                                     c_layers=C_LAYERS, vocab=VOCAB, vfeat_dim=VFEAT,
                                     max_frm_seq_len=MAX_FRM, weight_seed=WEIGHT_SEED,
                                     weight_std=WEIGHT_STD)),
           "state_dict_shapes": json.dumps(shapes),
           "num_subs": json.dumps(b["num_subs"]),
           "sub_idx2frame_idx": json.dumps(b["sub_idx2frame_idx"]),
           "grad_params": json.dumps(list(GRAD_PARAMS))}
    for k, v in b.items():
        if torch.is_tensor(v):
            out["b." + k] = v.numpy()
    with torch.no_grad():
        out["logits"] = model(batch(), "violin", compute_loss=False).numpy()
        out["loss"] = model(batch(), "violin", compute_loss=True).numpy()
    model.zero_grad()
    model(batch(), "violin", compute_loss=True).backward()
    params = dict(model.named_parameters())
    for n in GRAD_PARAMS:
        g = params[n].grad
        assert g is not None and float(g.abs().sum()) > 0, n
        out["g." + n] = g.numpy()
    dst = os.path.join(ROOT, "tests", "golden", "violin_tiny.npz")
    np.savez_compressed(dst, **out)
    print(f"violin_tiny.npz: {len(b['num_subs'])} rows, joint lengths {lens.tolist()}, "
          f"targets {b['targets'].view(-1).tolist()}, loss {float(out['loss']):.5f}")


if __name__ == "__main__":
    main()
