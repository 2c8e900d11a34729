"""Pretraining validation (evalpass.validate_pretrain, pretrain.py:387-608) against the reference's
own validate functions (tests/golden/pretrain_val_tiny.npz, written by
tools/gen_pretrain_val_golden.py), on a CPU with hero_b200.ops routed through
tests/fake_pretrain_val_ops.py. `run_fixture_comparison` is shared with the GPU test, which runs it
on the device with the kernels.

Tolerances: 2e-2 relative for losses and l2, 2e-2 of the cosine's range for the mean cosine
(near 0 on these random features); the encoder runs on bf16 operands, the reference in fp32. Hits are compared row by row where the reference's top-1 / top-2 logit gap
exceeds twice LOGIT_BOUND, the bf16 error bound of these small logits; a near-tie row may flip.
Stated deviation: a label exactly tied with another column for the row maximum counts as a hit
(the reference's torch.max reports one index of the tie); tests/test_pretrain_val_gpu.py pins it."""
import json

import numpy as np
import pytest
import torch

from tests import fake_pretrain_val_ops
from tests import golden_util as gu
from tests import pretrain_val_batches as pv

LOGIT_BOUND = 5e-2
RATE_KEYS = {"mlm": "tok_per_s", "mffr": "feat_per_s", "mfm-nce": "feat_per_s",
             "fom": "valid/ex_per_s", "vsm": "valid/ex_per_s"}


def build_model(tmp_path, fx, device="cpu"):
    from oracle import hero_oracle as orc
    from hero_b200.model import VideoModelConfig
    from hero_b200.pretrain import HeroForPretraining
    path = tmp_path / "pretrain_val.json"
    path.write_text(json.dumps(pv.model_json()))
    model = HeroForPretraining(VideoModelConfig(str(path)), vfeat_dim=pv.VFEAT,
                               max_frm_seq_len=pv.MAX_FRM, **pv.LOSS_WEIGHTS)
    shapes = json.loads(str(fx["param_shapes"]))
    missing, unexpected = model.load_state_dict(
        orc.seeded_weights(shapes, seed=pv.WEIGHT_SEED, std=pv.WEIGHT_STD), strict=False)
    assert not unexpected and not [k for k in missing if k in shapes], (missing, unexpected)
    with torch.no_grad():
        model.v_encoder.mask_embedding.weight[0].zero_()
    return model.to(device).train()


def loaders(device="cpu", attach=False):
    from hero_b200 import evalpass, synth
    from hero_b200.plan import attach_plan
    out = {}
    for task in pv.TASKS:
        batches = []
        for i in range(2):
            b = pv.batch(task, i)
            if attach:
                if task == "mlm":
                    evalpass.attach_mlm_plan(b)
                else:
                    attach_plan(b, "vsm" if task == "vsm" else "repr")
            batches.append(synth.to_device(b, device) if device != "cpu" else b)
        out[task] = batches
    return out


def run_fixture_comparison(tmp_path, ops_module, device="cpu", attach=False):
    """validate_pretrain on the fixture's batches (with host-built plans when `attach`: the MLM
    plan and FOM's host clip mask); returns nothing, asserts everything."""
    from hero_b200 import evalpass
    fx = gu.load("pretrain_val_tiny.npz")
    model = build_model(tmp_path, fx, device)
    hits = []
    real = ops_module.lm_head_ce_stats

    def spy(*a, **k):
        out = real(*a, **k)
        hits.append(out[2].cpu())
        return out

    ld = loaders(device, attach)
    kept = {task: [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in b.items()}
                   for b in bs] for task, bs in ld.items()}
    try:
        ops_module.lm_head_ce_stats = spy
        got = evalpass.validate_pretrain(model, ld, pv.Opts)
    finally:
        ops_module.lm_head_ce_stats = real
    assert model.training
    # the dict the reference logs: the same keys, values within tolerance
    want = {}
    for task in pv.TASKS:
        want.update({f"{task}_{k}": v for k, v in json.loads(str(fx["log." + task])).items()})
    assert set(got) == set(want) | {f"{t}_{k}" for t, k in RATE_KEYS.items()}
    for k, v in want.items():
        if k.endswith("acc"):
            continue
        scale = max(abs(v), 1.0) if k.endswith("cosine") else abs(v)    # cosine: range [-1, 1]
        assert abs(got[k] - v) <= 2e-2 * scale + 1e-6, (k, got[k], v)
    # hits: MLM and MFM-NCE row by row (spied in call order), FOM by count
    n_mlm = len(fx["hit.mlm"])
    rows = {"mlm": torch.cat(hits[:2]).numpy(), "mfm-nce": torch.cat(hits[2:]).numpy()}
    assert len(rows["mlm"]) == n_mlm and len(rows["mfm-nce"]) == len(fx["hit.mfm-nce"])
    for task, mine in rows.items():
        sure = fx["gap." + task] > 2 * LOGIT_BOUND
        assert sure.sum() >= len(sure) // 2
        assert np.array_equal(mine[sure].astype(bool), fx["hit." + task][sure]), task
        assert got[f"{task}_acc"] == pytest.approx(mine.sum() / len(mine))
    unsure = int((fx["gap.fom"] <= 2 * LOGIT_BOUND).sum())
    n_fom = len(fx["hit.fom"])
    assert abs(got["fom_valid/acc"] * n_fom - fx["hit.fom"].sum()) <= unsure + 1e-6
    # batches are not mutated, except forward_mfm's documented in-place zeroing of c_v_feats
    for task, bs in ld.items():
        for b, k0 in zip(bs, kept[task]):
            assert set(b) == set(k0), task
            for k, v in b.items():
                if torch.is_tensor(v) and not (task in ("mffr", "mfm-nce") and k == "c_v_feats"):
                    assert torch.equal(v, k0[k]), (task, k)


@pytest.mark.parametrize("attach", [False, True])
def test_validate_pretrain_matches_reference(tmp_path, monkeypatch, attach):
    from hero_b200 import ops
    fake_pretrain_val_ops.install(monkeypatch)
    run_fixture_comparison(tmp_path, ops, attach=attach)


def test_unknown_task_raises_and_restores_training(tmp_path, monkeypatch):
    from hero_b200 import evalpass
    fake_pretrain_val_ops.install(monkeypatch)
    model = build_model(tmp_path, gu.load("pretrain_val_tiny.npz"))
    with pytest.raises(ValueError, match="Undefined task"):
        evalpass.validate_pretrain(model, {"itm": []}, pv.Opts)
    assert model.training


@pytest.mark.parametrize("m, d", [(-1, 64), (4, 0), (4, 4353)])
def test_row_l2_cos_bounds_raise(m, d):
    from hero_b200 import ops
    with pytest.raises(ValueError):
        ops._row_stats_bounds("row_l2_cos", m, d)


class _StubMfm(torch.nn.Module):
    """Returns fixed predictions correlated with the batch's targets (cosine far from 0), so the
    wiring of validate_mffr / validate_mfm_nce into the row kernels is pinned row by row."""

    def __init__(self, pred, neg):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.pred, self.neg = pred, neg

    def forward(self, batch, task, compute_loss=False):
        return self.pred if task == "mffr" else (self.pred, self.neg)


def test_mffr_and_nce_wiring_with_correlated_predictions(monkeypatch):
    import torch.nn.functional as F
    from hero_b200 import evalpass
    fake_pretrain_val_ops.install(monkeypatch)
    g = torch.Generator().manual_seed(3)
    tgt = [torch.randn(n, 64, generator=g) for n in (5, 7)]
    pred = [2.0 * t + 0.5 * torch.randn(t.shape, generator=g) for t in tgt]
    neg = [torch.randn(9, 64, generator=g) for _ in tgt]
    l2 = torch.cat([(p - t).pow(2).sum(1).sqrt() for p, t in zip(pred, tgt)])
    cos = torch.cat([F.cosine_similarity(p, t, dim=-1) for p, t in zip(pred, tgt)])
    assert float(cos.mean()) > 0.8
    ce, hits = 0.0, 0
    for p, t, ng in zip(pred, tgt, neg):
        logits = torch.cat([p @ t.t(), p @ ng.t()], 1)
        lab = torch.arange(p.shape[0])
        ce += float(F.cross_entropy(logits, lab, reduction="sum"))
        hits += int((logits.argmax(-1) == lab).sum())
    n = l2.numel()
    for task, fn in (("mffr", evalpass.validate_mffr), ("mfm-nce", evalpass.validate_mfm_nce)):
        out = {}
        for i in range(2):
            m = _StubMfm(pred[i], neg[i])
            part = fn(m, [{"feat_targets": tgt[i]}])
            out[i] = part
        # two single-batch passes, combined with their row counts
        w = [tgt[0].shape[0], tgt[1].shape[0]]
        loss = sum(out[i]["loss"] * w[i] for i in range(2)) / n
        cosine = sum(out[i]["cosine"] * w[i] for i in range(2)) / n
        assert cosine == pytest.approx(float(cos.mean()), rel=1e-5)
        if task == "mffr":
            assert loss == pytest.approx(float(l2.mean()), rel=1e-5)
        else:
            assert out[0]["l2"] * w[0] + out[1]["l2"] * w[1] == pytest.approx(float(l2.sum()),
                                                                            rel=1e-5)
            # bf16 operands in the NCE GEMM (the fake rounds them as the kernel does)
            assert loss == pytest.approx(ce / n, rel=2e-2)
            assert round(sum(out[i]["acc"] * w[i] for i in range(2))) == hits
