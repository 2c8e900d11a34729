"""Writes tests/golden/pretrain_val_tiny.npz: the reference's own pretraining validation
(pretrain.py validate_mlm / _mffr / _mfm_nce / _fom / _vsm) on its HeroForPretraining in fp32 on
the CPU, eval mode, tiny configuration (tests/pretrain_val_batches.py: H 128, vocabulary 120, 64-d
frame features), two synthetic batches per task.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_pretrain_val_golden.py

The reference's functions are imported from its checkout and run unchanged; only
`all_gather_list` is replaced by `lambda x: [x]` (one process). `oracle.gen_golden`'s
check_collate_layout first confirms that hero_b200.synth.video_batch reproduces the reference's
video_collate layout (on its own two-clip spec); the task-specific masking of the synthetic
batches (txt_mask_tgt / txt_labels, c_v_masks / feat_targets, shuffled_orders / targets, the VSM
query fields) is not checked against the reference's task collates. Weights are
`oracle.hero_oracle.seeded_weights` over the reference's parameter shapes (stored, so the tests
rebuild them). Stored: every returned dict without its `*_per_s` rate, and per row of MLM,
MFM-NCE and FOM (valid rows) the gap between the top-1 and top-2 logits and whether the reference
counted a hit, so tests compare hits only where a hit means something.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden as gg  # noqa: E402
from oracle import hero_oracle as orc  # noqa: E402
from tests import pretrain_val_batches as pv  # noqa: E402


def build():
    from model.model import VideoModelConfig
    from model.pretrain import HeroForPretraining
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(pv.model_json(), f)
        path = f.name
    config = VideoModelConfig(path)
    os.unlink(path)
    model = HeroForPretraining(config, vfeat_dim=pv.VFEAT, max_frm_seq_len=pv.MAX_FRM,
                               **pv.LOSS_WEIGHTS)
    shapes = {k: list(p.shape) for k, p in model.named_parameters()}
    missing, unexpected = model.load_state_dict(
        orc.seeded_weights(shapes, seed=pv.WEIGHT_SEED, std=pv.WEIGHT_STD), strict=False)
    assert not unexpected and not [k for k in missing if k in shapes], (missing, unexpected)
    with torch.no_grad():
        model.v_encoder.mask_embedding.weight[0].zero_()          # padding row
    return model.eval(), shapes


def gap_hit(scores, labels):
    top2 = scores.float().topk(2, dim=-1).values
    return (top2[:, 0] - top2[:, 1]).numpy(), (scores.max(dim=-1)[1] == labels).numpy()


def row_gaps(model, task):
    """Per row (top-1 - top-2 logit gap, reference hit) over both batches of `task`."""
    out = []
    with torch.no_grad():
        for i in range(2):
            b = pv.batch(task, i)
            if task == "mlm":
                out.append(gap_hit(model(b, task="mlm", compute_loss=False), b["txt_labels"]))
            elif task == "mfm-nce":
                feats, neg = model(b, task="mfm-nce", compute_loss=False)
                logits = model.v_encoder.mfm_nce(feats, b["feat_targets"], neg, compute_loss=False)
                out.append(gap_hit(logits, torch.arange(logits.shape[0])))
            elif task == "fom":
                tg = b.pop("targets").reshape(-1)
                b.pop("vids")
                scores = model(b, task="fom", compute_loss=False)
                out.append(gap_hit(scores[tg != -1], tg[tg != -1]))
    return (np.concatenate([g for g, _ in out]), np.concatenate([h for _, h in out]))


def main():
    gg.install_stubs()
    gg.check_collate_layout()
    import pretrain
    pretrain.all_gather_list = lambda x: [x]
    model, shapes = build()
    fns = {"mlm": pretrain.validate_mlm, "mffr": pretrain.validate_mffr,
           "mfm-nce": pretrain.validate_mfm_nce, "fom": pretrain.validate_fom,
           "vsm": lambda m, loader: pretrain.validate_vsm(m, loader, pv.Opts)}
    out = {"config": json.dumps(dict(model_json=pv.model_json(), vfeat_dim=pv.VFEAT,
                                     max_frm_seq_len=pv.MAX_FRM, weight_seed=pv.WEIGHT_SEED,
                                     weight_std=pv.WEIGHT_STD, loss_weights=pv.LOSS_WEIGHTS,
                                     seeds=pv.SEEDS)),
           "param_shapes": json.dumps(shapes)}
    for task in pv.TASKS:
        with torch.no_grad():
            log = fns[task](model, [pv.batch(task, i) for i in range(2)])
        log = {k: float(v) for k, v in log.items() if not k.endswith("per_s")}
        out["log." + task] = json.dumps(log)
        if task in ("mlm", "mfm-nce", "fom"):
            out["gap." + task], out["hit." + task] = row_gaps(model, task)
            assert int(out["hit." + task].sum()) == round(log.get("acc", log.get("valid/acc")) *
                                                          len(out["hit." + task]))
        print(task, log)
    dst = os.path.join(ROOT, "tests", "golden", "pretrain_val_tiny.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst)


if __name__ == "__main__":
    main()
