"""Prints error statistics of the CUDA encoder vs the CPU oracle / reference goldens (used to
choose and justify the tolerances written in tests/test_encoder_gpu.py). Lives under tests/
because it calls the oracle (test infrastructure); run as `python tests/parity_report.py` on a GPU
box. Not collected by pytest (no test_ prefix)."""
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from hero_b200 import synth
from hero_b200.model import HierarchicalVlModel, VideoModelConfig
from oracle import hero_oracle as orc
from tests import golden_util as gu


def build(d, P):
    def cfg(n, v):
        c = {"attention_probs_dropout_prob": 0.1, "hidden_act": "gelu", "hidden_dropout_prob": 0.1,
             "hidden_size": d["hidden"], "initializer_range": 0.02, "intermediate_size": d["inter"],
             "max_position_embeddings": 514, "num_attention_heads": d["heads"],
             "num_hidden_layers": n, "type_vocab_size": 2}
        if v:
            c["vocab_size"] = d["vocab"]
        return c
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "m.json")
        json.dump({"f_config": cfg(d["f_layers"], True), "c_config": cfg(d["c_layers"], False)},
                  open(p, "w"))
        m = HierarchicalVlModel(VideoModelConfig(p), vfeat_dim=d["vfeat_dim"],
                                max_frm_seq_len=d["max_img_len"])
    m.load_state_dict(P, strict=False)
    return m.cuda().eval()


def stats(got, ref, mask):
    got = got.detach().float().cpu().numpy()[mask]
    ref = np.asarray(ref)[mask]
    err = np.abs(got - ref)
    cos = (got * ref).sum(-1) / (np.linalg.norm(got, axis=-1) * np.linalg.norm(ref, axis=-1))
    return {"max": float(err.max()), "mean": float(err.mean()), "p999": float(np.quantile(err, 0.999)),
            "min_cos": float(cos.min()), "ref_absmax": float(np.abs(ref).max())}


def bf16_torch_reference(P, vb, d):
    """Same oracle arithmetic with weights/activations rounded to bf16 at layer boundaries is not
    available; instead report the oracle run under torch CPU bfloat16 autocast as a yardstick."""
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = orc.hierarchical_repr(P, vb, d["f_layers"], d["c_layers"], d["heads"])
    return out.float()


def main():
    rep = {}
    fx = gu.load("hier_full_small.npz")
    d = gu.dims_of(fx)
    P = gu.weights_for(fx)
    vb, qb = gu.full_small_batches(fx)
    model = build(d, P)
    with torch.no_grad():
        clip = model(synth.to_device(vb, "cuda"), "repr")
        q = model.f_encoder(synth.to_device(qb, "cuda"), "txt")[0]
    m = vb["c_attn_masks"].bool().numpy()
    rep["full_depth_clip"] = stats(clip, fx["clip_out"], m)
    rep["full_depth_query"] = stats(q, fx["q_seq_out"], qb["attn_masks"].bool().numpy())
    rep["full_depth_clip_cpu_bf16_autocast"] = stats(bf16_torch_reference(P, vb, d), fx["clip_out"], m)
    del model

    d2 = dict(hidden=768, inter=3072, heads=12, f_layers=2, c_layers=1, vocab=50272,
              vfeat_dim=4352, max_img_len=100)
    P = orc.seeded_weights(orc.param_shapes(f_layers=2, c_layers=1), seed=5)
    for kind in ("ragged", "dense"):
        if kind == "ragged":
            vb, qb = synth.syn_tvr_ragged(batch_size=4, seed=99, t_range=(20, 40), s_range=(4, 8),
                                          l_range=(4, 30), q_range=(6, 20))
        else:
            vb, qb = synth.syn_tvr_dense(batch_size=2, seed=7)
        g = torch.Generator().manual_seed(1)
        w1 = torch.randn(vb["c_v_feats"].shape[0], vb["c_v_feats"].shape[1], 768, generator=g)
        w1 = w1 * vb["c_attn_masks"].unsqueeze(-1)
        w2 = torch.randn(qb["input_ids"].shape[0], qb["input_ids"].shape[1], 768, generator=g)
        w2 = w2 * qb["attn_masks"].unsqueeze(-1)
        Pg = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        clip_ref = orc.hierarchical_repr(Pg, vb, 2, 1, 12)
        q_ref = orc.cross_modal_txt(Pg, "f_encoder.", qb, 2, 12)
        ((clip_ref * w1).sum() + (q_ref * w2).sum()).backward()
        model = build(d2, P)
        clip = model(synth.to_device(vb, "cuda"), "repr")
        q = model.f_encoder(synth.to_device(qb, "cuda"), "txt")[0]
        ((clip * w1.cuda()).sum() + (q * w2.cuda()).sum()).backward()
        rep[kind + "_clip"] = stats(clip, clip_ref.detach().numpy(), vb["c_attn_masks"].bool().numpy())
        rep[kind + "_query"] = stats(q, q_ref.detach().numpy(), qb["attn_masks"].bool().numpy())
        named = dict(model.named_parameters())
        rel = {}
        for k, v in Pg.items():
            if v.grad is None or "pooler" in k or "mask_embedding" in k:
                continue
            got = named[k].grad
            if got is None:
                rel[k] = "MISSING"
                continue
            den = v.grad.norm().item()
            rel[k] = round((got.float().cpu() - v.grad).norm().item() / max(den, 1e-12), 5)
        worst = sorted(((v, k) for k, v in rel.items() if not isinstance(v, str)), reverse=True)[:15]
        rep[kind + "_grad_worst"] = worst
        rep[kind + "_grad_missing"] = [k for k, v in rel.items() if isinstance(v, str)]
        del model
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
