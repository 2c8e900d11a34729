"""Writes tests/golden/videoqa_tiny.npz: the reference's HeroForVideoQA (model/videoQA.py) on a
tiny configuration and a ragged TVQA-style batch.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_videoqa_golden.py

Configuration: H = 128, 2 heads, 2 cross-modal + 2 temporal layers, vocabulary 120, 64-d frame
features. Weights are `oracle.hero_oracle.seeded_weights` over the reference's state_dict shapes
(seed WEIGHT_SEED; rebuilt by the tests from the stored shape list), model in eval mode;
the batch is `hero_b200.synth.syn_videoqa_batch` with 3 videos x 5 candidates, ragged clips, one
video without a target and one without start / end targets, and joint [frames | QA] rows longer
than 128 tokens. Stored: the batch, the reference's state_dict key / shape list, the
logits and both losses for "tvqa" and "how2qa", and the gradients of qa_loss + 0.4 * temporal_loss
for the parameters listed in GRAD_PARAMS (every head parameter except the two biases in front
of each softmax whose gradient is zero in exact arithmetic: both softmaxes are shift-invariant).
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
WEIGHT_SEED, WEIGHT_STD = 7, 0.1   # std 0.1: the candidates of a video differ visibly
LW_ST_ED = 0.4
GRAD_PARAMS = (
    "qa_pool.weight", "st_ed_pool.weight",
    "qa_pred_head.linear_1.weight", "qa_pred_head.linear_1.bias",
    "qa_pred_head.LayerNorm.weight", "qa_pred_head.linear_2.weight",
    "st_ed_pred_head.linear_1.weight", "st_ed_pred_head.linear_1.bias",
    "st_ed_pred_head.LayerNorm.weight", "st_ed_pred_head.linear_2.weight",
    "v_encoder.c_encoder.encoder.layer.0.attention.self.query.weight",
    "v_encoder.c_encoder.encoder.layer.0.attention.self.key.weight",
    "v_encoder.c_encoder.encoder.layer.0.attention.self.value.weight",
    "v_encoder.c_encoder.embeddings.position_embeddings.weight",
    "v_encoder.f_encoder.embeddings.word_embeddings.weight",
    "v_encoder.f_encoder.encoder.layer.0.output.dense.weight",
)


def batch():
    return synth.syn_videoqa_batch(n_videos=3, n_cand=5, seed=1, t_range=(6, 110),
                                   s_range=(2, 5), l_range=(3, 10), qa_range=(20, 60),
                                   vfeat_dim=VFEAT, vocab=VOCAB, no_target=(1,), no_ts=(2,))


def main():
    gg.install_stubs()
    from model.model import VideoModelConfig
    from model.videoQA import HeroForVideoQA
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(gg.model_json(H, INTER, HEADS, F_LAYERS, C_LAYERS, VOCAB), f)
        path = f.name
    config = VideoModelConfig(path)
    os.unlink(path)
    model = HeroForVideoQA(config, vfeat_dim=VFEAT, max_frm_seq_len=MAX_FRM).eval()
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(orc.seeded_weights(shapes, seed=WEIGHT_SEED, std=WEIGHT_STD))
    b = batch()
    lens = b["c_attn_masks"].sum(1) + b["qa_attn_masks"].sum(1)
    assert int(lens.max()) > 128 and int(lens.min()) <= 128, lens
    out = {"config": json.dumps(dict(hidden=H, inter=INTER, heads=HEADS, f_layers=F_LAYERS,
                                     c_layers=C_LAYERS, vocab=VOCAB, vfeat_dim=VFEAT,
                                     max_frm_seq_len=MAX_FRM, lw_st_ed=LW_ST_ED,
                                     weight_seed=WEIGHT_SEED, weight_std=WEIGHT_STD)),
           "state_dict_shapes": json.dumps(shapes),
           "num_subs": json.dumps(b["num_subs"]),
           "sub_idx2frame_idx": json.dumps(b["sub_idx2frame_idx"]),
           "grad_params": json.dumps(list(GRAD_PARAMS))}
    for k, v in b.items():
        if torch.is_tensor(v):
            out["b." + k] = v.numpy()
    with torch.no_grad():
        for task in ("tvqa", "how2qa"):
            out[f"{task}.logits"] = model(batch(), task, compute_loss=False).numpy()
            qa_loss, temporal_loss = model(batch(), task, compute_loss=True)
            out[f"{task}.qa_loss"] = qa_loss.numpy()
            out[f"{task}.temporal_loss"] = temporal_loss.numpy()
    model.zero_grad()
    qa_loss, temporal_loss = model(batch(), "tvqa", compute_loss=True)
    (qa_loss + LW_ST_ED * temporal_loss).backward()
    params = dict(model.named_parameters())
    for n in GRAD_PARAMS:
        out["g." + n] = params[n].grad.numpy()
    dst = os.path.join(ROOT, "tests", "golden", "videoqa_tiny.npz")
    np.savez_compressed(dst, **out)
    print(f"videoqa_tiny.npz: {len(b['num_subs'])} rows, joint lengths {lens.tolist()}, "
          f"qa_loss {float(out['tvqa.qa_loss']):.5f}, "
          f"temporal_loss {float(out['tvqa.temporal_loss']):.5f}")


if __name__ == "__main__":
    main()
