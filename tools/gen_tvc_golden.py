"""Writes tests/golden/tvc_tiny.npz: the reference's HeroForTvc (model/tvc.py) on the tiny
configuration of tests/golden/violin_tiny.npz plus a 2-layer decoder, on a ragged TVC batch.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_tvc_golden.py

It first checks that `hero_b200.synth.syn_tvc_batch` equals the reference's own
TvcTrainDataset.collate and TvcValDataset.collate (data/tvc.py:140-218) applied to the same
dataset items, built the way the datasets' __getitem__ builds them.

Configuration: H = 128, 2 heads, 2 cross-modal + 2 temporal + 2 decoder layers, vocabulary 120,
64-d frame features, decoder position table 1024. Weights are `oracle.hero_oracle.seeded_weights`
over the reference's parameter shapes (seed WEIGHT_SEED; the two buffers `decoder.tri_mask` and
`loss_func.one_hot` keep their constructed values), model in fp32 on the CPU in eval mode. The
batch is 3 videos with 2-6 caption segments each, one of them empty (st == ed == nframes).
Stored: the batch, the state_dict key / shape list, the teacher-forced logits, the per-token loss
vectors with lsr 0.1 and lsr 0, and from TvcGenerator.greedy_decode with max_step 12 the greedy
ids of every position (uncut; the cut lists are checked against them here) and the gap between
the top-1 and top-2 logits at every decoded position.
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

H, INTER, HEADS, F_LAYERS, C_LAYERS, D_LAYERS, VOCAB = 128, 256, 2, 2, 2, 2, 120
VFEAT, MAX_FRM, D_MAX_POS = 64, 120, 1024
WEIGHT_SEED, WEIGHT_STD = 7, 0.1
MAX_STEP = 12
BUFFERS = ("decoder.tri_mask", "loss_func.one_hot")
BATCH_ARGS = dict(n_videos=3, seed=21, t_range=(6, 60), s_range=(2, 5), l_range=(3, 10),
                  seg_range=(2, 6), c_range=(4, 14), n_empty=1, vfeat_dim=VFEAT, vocab=VOCAB)


def model_json():
    j = gg.model_json(H, INTER, HEADS, F_LAYERS, C_LAYERS, VOCAB)
    d = dict(j["f_config"], num_hidden_layers=D_LAYERS, max_position_embeddings=D_MAX_POS,
             type_vocab_size=1)
    j["d_config"] = d
    return j


def batch(split="train"):
    return synth.syn_tvc_batch(**BATCH_ARGS, split=split)


def video_inputs(c):
    """VideoFeatSubTokDataset.__getitem__ (data/data.py:346-397) for one synthetic clip."""
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
    return (ids, feats, masks, c["feats"], torch.tensor([1] * T), len(c["subs"]),
            c["sub2frames"])


def check_tvc_collates():
    from data.tvc import TvcTrainDataset, TvcValDataset
    keys = ("f_sub_input_ids", "f_sub_pos_ids", "f_v_feats", "f_v_pos_ids", "f_attn_masks",
            "f_gather_index", "c_v_feats", "c_attn_masks", "cap_attn_mask")
    for args in (BATCH_ARGS, dict(BATCH_ARGS, n_videos=4, seed=5)):
        items = synth.syn_tvc_items(**args)
        train = TvcTrainDataset.collate([
            (video_inputs(it["clip"]), it["clip_ranges"],
             [(i, t, torch.tensor([1] * (ed - st))) for i, t, (st, ed)
              in zip(it["input_ids"], it["tgt_ids"], it["clip_ranges"])]) for it in items])
        val = TvcValDataset.collate([
            (video_inputs(it["clip"]), it["clip_ranges"],
             [torch.tensor([1] * (ed - st)) for st, ed in it["clip_ranges"]],
             (it["vid"], it["clip_ids"], it["ts"], [f"caption {c}" for c in it["clip_ids"]]))
            for it in items])
        for ref, split, extra in ((train, "train", ("cap_input_ids", "cap_pos_ids", "cap_tgt_ids")),
                                  (val, "val", ())):
            mine = synth.syn_tvc_batch(**args, split=split)
            for k in keys + extra:
                assert torch.equal(ref[k], mine[k]), (split, k)
            for k in ("clip_ranges", "num_subs", "sub_idx2frame_idx") + (
                    ("vid_names", "clip_ids", "all_ts", "gts") if split == "val" else ()):
                assert ref[k] == mine[k], (split, k)
    print("syn_tvc_batch == reference TvcTrainDataset.collate / TvcValDataset.collate")


def build(lsr):
    from model.model import VideoModelConfig
    from model.tvc import HeroForTvc
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(model_json(), f)
        path = f.name
    config = VideoModelConfig(path)
    os.unlink(path)
    model = HeroForTvc(config, vfeat_dim=VFEAT, max_frm_seq_len=MAX_FRM, lsr=lsr).eval()
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    params = {k: s for k, s in shapes.items() if k not in BUFFERS}
    missing, unexpected = model.load_state_dict(
        orc.seeded_weights(params, seed=WEIGHT_SEED, std=WEIGHT_STD), strict=False)
    assert not unexpected and set(missing) <= set(BUFFERS), (missing, unexpected)
    return model, shapes


def greedy(model):
    """TvcGenerator.greedy_decode with .cuda() as the identity; returns (cut lists, the scores of
    its last full decoder pass)."""
    from model.tvc import TvcGenerator
    last = {}
    decode = model.decode

    def spy(*a, **kw):
        last["score"] = decode(*a, **kw)
        return last["score"]

    model.decode = spy
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **kw: self
    try:
        gen = TvcGenerator(model, MAX_STEP, synth.BOS, synth.EOS, fp16=False)
        with torch.no_grad():
            out = gen.greedy_decode(batch("val"))
    finally:
        torch.Tensor.cuda = cuda
        del model.decode
    return gen, out, last["score"]


def main():
    gg.install_stubs()
    check_tvc_collates()
    model, shapes = build(0.1)
    model0, shapes0 = build(0.0)
    b = batch()
    empty = [i for i, (st, ed) in enumerate(r for rs in b["clip_ranges"] for r in rs) if st == ed]
    assert len(empty) == 1, empty
    out = {"config": json.dumps(dict(hidden=H, inter=INTER, heads=HEADS, f_layers=F_LAYERS,
                                     c_layers=C_LAYERS, d_layers=D_LAYERS, vocab=VOCAB,
                                     vfeat_dim=VFEAT, max_frm_seq_len=MAX_FRM,
                                     d_max_pos=D_MAX_POS, weight_seed=WEIGHT_SEED,
                                     weight_std=WEIGHT_STD, max_step=MAX_STEP,
                                     buffers=list(BUFFERS), batch_args=BATCH_ARGS)),
           "state_dict_shapes": json.dumps(shapes),
           "state_dict_shapes_lsr0": json.dumps(shapes0),
           "clip_ranges": json.dumps(b["clip_ranges"]),
           "num_subs": json.dumps(b["num_subs"]),
           "sub_idx2frame_idx": json.dumps(b["sub_idx2frame_idx"])}
    for k, v in b.items():
        if torch.is_tensor(v):
            out["b." + k] = v.numpy()
    with torch.no_grad():
        out["logits"] = model(batch(), compute_loss=False).numpy()
        out["loss_lsr"] = model(batch(), compute_loss=True).numpy()
        out["loss_ce"] = model0(batch(), compute_loss=True).numpy()
    gen, cut, score = greedy(model)
    top2 = score.topk(2, dim=-1).values
    ids = score.max(dim=-1)[1]
    assert [gen.cut_eos(r) for r in ids.tolist()] == cut
    out["greedy_ids"] = ids.numpy().astype(np.int64)
    out["greedy_gap"] = (top2[..., 0] - top2[..., 1]).numpy()
    dst = os.path.join(ROOT, "tests", "golden", "tvc_tiny.npz")
    np.savez_compressed(dst, **out)
    print(f"tvc_tiny.npz: {b['cap_input_ids'].shape[0]} captions of {b['cap_input_ids'].shape[1]} "
          f"positions, empty segment {empty}, greedy lengths {[len(c) for c in cut]}, "
          f"min gap {float(out['greedy_gap'].min()):.2e}")


if __name__ == "__main__":
    main()
