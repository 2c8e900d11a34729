"""Pins the CPU oracle against outputs of the unmodified reference (tests/golden/*.npz, produced
by oracle/gen_golden.py from the reference). fp32 on both sides -> tight tolerance."""
import numpy as np
import torch

from oracle import hero_oracle as orc
from tests import golden_util as gu
from hero_b200 import synth


def _assert_close(got, ref, tol=2e-5, what=""):
    got = got.detach().numpy() if torch.is_tensor(got) else got
    err = np.abs(got - ref).max()
    scale = max(1.0, np.abs(ref).max())
    assert err <= tol * scale, f"{what}: max abs err {err} (scale {scale})"


def test_tiny_hierarchical_forward_matches_reference():
    fx = gu.load("hier_tiny.npz")
    d = gu.dims_of(fx)
    P = gu.weights_for(fx)
    vb, qb = gu.stored_batches(fx)
    f_seq = orc.cross_modal_repr(P, "f_encoder.", vb, d["f_layers"], d["heads"])
    m = vb["f_attn_masks"].bool().numpy()
    _assert_close(f_seq.numpy()[m], fx["f_seq_out"][m], what="f_encoder sequence output (valid)")
    # padded positions too: the oracle mirrors the reference's padded arithmetic exactly
    _assert_close(f_seq, fx["f_seq_out"], what="f_encoder sequence output (all)")
    _assert_close(orc.pooler(P, "f_encoder.pooler.", f_seq), fx["f_pooled"], what="pooler")
    clip = orc.hierarchical_repr(P, vb, d["f_layers"], d["c_layers"], d["heads"])
    _assert_close(clip, fx["clip_out"], what="clip outputs")
    pre = orc.hierarchical_repr(P, vb, d["f_layers"], d["c_layers"], d["heads"], encode_clip=False)
    _assert_close(pre, fx["pre_clip"], what="pre-temporal features")
    q = orc.cross_modal_txt(P, "f_encoder.", qb, d["f_layers"], d["heads"])
    _assert_close(q, fx["q_seq_out"], what="query rows")


def test_tiny_hierarchical_gradients_match_reference():
    fx = gu.load("hier_tiny.npz")
    d = gu.dims_of(fx)
    P = {k: v.clone().requires_grad_(True) for k, v in gu.weights_for(fx).items()}
    vb, qb = gu.stored_batches(fx)
    clip = orc.hierarchical_repr(P, vb, d["f_layers"], d["c_layers"], d["heads"])
    q = orc.cross_modal_txt(P, "f_encoder.", qb, d["f_layers"], d["heads"])
    loss = (clip * torch.from_numpy(fx["loss_w1"])).sum() + (q * torch.from_numpy(fx["loss_w2"])).sum()
    assert abs(loss.item() - float(fx["loss"])) < 1e-3
    loss.backward()
    for k, ref in fx.items():
        if not k.startswith("grad."):
            continue
        g = P[k[5:]].grad
        assert g is not None, k
        _assert_close(g, ref, tol=1e-4, what=k)


def test_config1_real_dims_matches_reference():
    fx = gu.load("xm1_config1.npz")
    d = gu.dims_of(fx)
    P = gu.weights_for(fx)
    xb = synth.syn_xm_1(seed=int(fx["seed_batch"]))
    seq = orc.cross_modal_repr(P, "f_encoder.", xb, d["f_layers"], d["heads"])
    _assert_close(seq, fx["seq_out"], tol=5e-5, what="config-1 sequence output")
    _assert_close(orc.pooler(P, "f_encoder.pooler.", seq), fx["pooled"], tol=5e-5, what="pooled")


def test_full_depth_small_batch_matches_reference():
    fx = gu.load("hier_full_small.npz")
    d = gu.dims_of(fx)
    P = gu.weights_for(fx)
    vb, qb = gu.full_small_batches(fx)
    assert np.array_equal(vb["c_attn_masks"].numpy(), fx["c_attn_masks"])
    clip = orc.hierarchical_repr(P, vb, d["f_layers"], d["c_layers"], d["heads"])
    _assert_close(clip, fx["clip_out"], tol=1e-4, what="full-depth clip outputs")
    q = orc.cross_modal_txt(P, "f_encoder.", qb, d["f_layers"], d["heads"])
    _assert_close(q, fx["q_seq_out"], tol=1e-4, what="full-depth query rows")


def test_adamw_matches_reference_trajectory():
    fx = gu.load("adamw.npz")
    p = torch.from_numpy(fx["p0"]).clone()
    m = torch.zeros_like(p)
    v = torch.zeros_like(p)
    for t, g in enumerate(fx["grads"], start=1):
        p, m, v = orc.adamw_step(p, torch.from_numpy(g), m, v, t, float(fx["lr"]), float(fx["beta1"]),
                                 float(fx["beta2"]), float(fx["eps"]), float(fx["weight_decay"]))
        _assert_close(p, fx["traj"][t - 1], tol=1e-6, what=f"adamw step {t}")
