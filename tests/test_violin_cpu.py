"""HeroForViolin (model/violin.py) against the unmodified reference on a tiny configuration
(tests/golden/violin_tiny.npz, written by tools/gen_violin_golden.py), with hero_b200.ops routed
through tests/fake_violin_ops.py: the VIOLIN plan, the model, PlanPool transport and the
evaluation loop on the host. The CUDA kernels are covered by test_violin_gpu.py."""
import json

import numpy as np
import pytest
import torch

from oracle import hero_oracle as orc
from tests import fake_violin_ops
from tests import golden_util as gu
from tests import test_videoqa_cpu as qa


def fixture():
    return gu.load("violin_tiny.npz")


def violin_model(tmp_path, vx):
    from hero_b200.model import VideoModelConfig
    from hero_b200.violin import HeroForViolin
    from oracle import gen_golden as gg
    c = json.loads(str(vx["config"]))
    path = tmp_path / "violin.json"
    path.write_text(json.dumps(gg.model_json(c["hidden"], c["inter"], c["heads"], c["f_layers"],
                                             c["c_layers"], c["vocab"])))
    model = HeroForViolin(VideoModelConfig(str(path)), vfeat_dim=c["vfeat_dim"],
                          max_frm_seq_len=c["max_frm_seq_len"])
    shapes = json.loads(str(vx["state_dict_shapes"]))
    model.load_state_dict(orc.seeded_weights(shapes, seed=c["weight_seed"], std=c["weight_std"]))
    return model.eval()


def test_state_dict_keys_and_shapes_match_reference(tmp_path):
    vx = fixture()
    ref = json.loads(str(vx["state_dict_shapes"]))
    ours = {k: list(v.shape) for k, v in violin_model(tmp_path, vx).state_dict().items()}
    assert ours == ref


@pytest.mark.parametrize("attach", [False, True])
def test_logits_loss_and_gradients_match_reference(tmp_path, monkeypatch, attach):
    from hero_b200.plan import attach_plan
    fake_violin_ops.install(monkeypatch)
    vx = fixture()
    model = violin_model(tmp_path, vx)

    def batch():
        b = qa.qa_batch(vx)
        return attach_plan(b, kind="violin") if attach else b

    with torch.no_grad():
        logits = model(batch(), "violin", compute_loss=False)
        loss = model(batch())
    ref = vx["logits"]
    assert logits.shape == ref.shape == (6, 1)
    assert np.abs(logits.numpy() - ref).max() <= 2e-2 * max(np.abs(ref).max(), 1.0)
    assert abs(float(loss) - float(vx["loss"])) < 2e-2
    model(batch(), "violin").backward()
    params = dict(model.named_parameters())
    for name in json.loads(str(vx["grad_params"])):
        ref = torch.from_numpy(vx["g." + name])
        got = params[name].grad
        assert got is not None, name
        rel = float((got - ref).norm() / ref.norm().clamp(min=1e-12))
        assert rel < 3e-2, (name, rel)


def test_unknown_task_raises(tmp_path, monkeypatch):
    fake_violin_ops.install(monkeypatch)
    vx = fixture()
    model = violin_model(tmp_path, vx)
    for task in ("tvqa", "how2qa", "vcmr"):
        with pytest.raises(ValueError, match="Unrecognized task"):
            model(qa.qa_batch(vx), task)


def test_single_pool_bounds_raise_before_launch():
    from hero_b200 import functional as Fn
    for nv, length, h in ((1, 513, 16), (1, 4, 12), (0, 4, 16)):
        fmap = torch.full((max(nv, 1) * length,), -1, dtype=torch.int32)
        with pytest.raises(ValueError):
            Fn.qa_pool(torch.zeros(4, h), torch.zeros(1, h), None, fmap,
                       torch.zeros(fmap.numel()), nv, 1, length)


def test_violin_plan_single_candidate_ragged_and_long_rows():
    """Every statement row is its own 'video' (Nq = 1) and pools over its own frames; a row of
    more than 128 tokens takes the long-row attention tiles."""
    from hero_b200.plan import ATTN_TILE, qa_plan, video_kind
    c = torch.zeros(4, 6, dtype=torch.long)
    c[0, :6], c[1, :6], c[2, :1], c[3, :1] = 1, 1, 1, 1         # two videos, two statements each
    q = torch.zeros(4, 130, dtype=torch.long)
    q[0, :5], q[1, :130], q[2, :2], q[3, :7] = 1, 1, 1, 1
    ids = torch.arange(4 * 130).view(4, 130) + 3
    b = {"c_attn_masks": c, "q_attn_masks": q, "q_input_ids": ids,
         "q_pos_ids": torch.arange(130).unsqueeze(0), "targets": torch.tensor([[1], [0], [0], [1]])}
    assert video_kind(b) == "violin"
    p = qa_plan(b, "q")
    assert (p.n_videos, p.n_cand, p.length) == (4, 1, 6)
    lens = [11, 136, 3, 8]
    assert p.seq.lens.tolist() == lens
    assert p.seq.n_long == p.n_long_rows == 1 and p.seq.max_long == 136 > ATTN_TILE
    starts = np.cumsum([0] + lens)
    fmap = p.frame_map.reshape(4, 6)
    for r, n in enumerate((6, 6, 1, 1)):
        assert fmap[r, :n].tolist() == list(range(starts[r], starts[r] + n))
        assert (fmap[r, n:] == -1).all()
    assert p.qa_ids[:5].tolist() == ids[0, :5].tolist()
    assert p.qa_pos[5:135].tolist() == list(range(130))
    # CSR of the position-table gradients lists every frame k under its temporal position
    off, idx = p.cpos_off, p.cpos_idx
    assert sorted(idx[off[0]:off[1]].tolist()) == [0, 6, 12, 13]


def test_plan_pool_inputs_carry_the_violin_plan():
    """plan_inputs / build_plans (what a PlanPool worker runs) and PlanPool.attach give a VIOLIN
    batch the same plans that attach_plan(kind="violin") builds in process."""
    from hero_b200.plan import (PLAN_KEY, QA_PLAN_KEY, PlanPool, attach_plan, build_plans,
                                plan_inputs, video_kind)
    b = qa.qa_batch(fixture())
    assert video_kind(b) == "violin"

    class Done:
        def result(self):
            return build_plans(plan_inputs(b, "violin"))

    pooled, _ = PlanPool.attach(Done(), dict(b))
    direct = attach_plan(dict(b), kind="violin")
    assert "_qa" not in pooled[PLAN_KEY].__dict__
    p, q = pooled[QA_PLAN_KEY], direct[QA_PLAN_KEY]
    assert (q.n_videos, q.n_cand) == (6, 1)
    for name in ("frame_map", "frm_tok", "frm_t", "qa_tok", "qa_ids", "qa_pos", "cpos_off",
                 "cpos_idx", "qpos_off", "qpos_idx"):
        assert np.array_equal(getattr(p, name), getattr(q, name)), name
    assert np.array_equal(p.seq.tile_tok0, q.seq.tile_tok0) and p.seq.n_long == q.seq.n_long == 1


def _host_validate_violin(batches, save_logits):
    """eval_violin.py:118-164 restated on the host, for batches of at least two rows (the
    reference's `predictions.squeeze().cpu().tolist()` is an int for one row)."""
    F = torch.nn.functional
    val_loss, n_ex, tot_score, results, logits = 0.0, 0, 0, {}, {}
    for qids, scores, targets in batches:
        predictions = (torch.sigmoid(scores) > 0.5).long()
        for qid, answer in zip(qids, predictions.squeeze().tolist()):
            results[str(qid)] = answer
        if save_logits:
            for qid, logit in zip(qids, scores.tolist()):
                logits[str(qid)] = logit
        val_loss += F.binary_cross_entropy(torch.sigmoid(scores), targets.to(scores.dtype),
                                           reduction="sum").item()
        tot_score += (predictions.squeeze() == targets.squeeze()).sum().item()
        n_ex += len(qids)
    return val_loss / n_ex, tot_score / n_ex, results, logits


class _Fixed(torch.nn.Module):
    def __init__(self, scores):
        super().__init__()
        self.scores, self.i = scores, 0

    def forward(self, batch, task, compute_loss=False):
        assert task == "violin" and not compute_loss
        s = self.scores[self.i]
        self.i += 1
        return s


def test_validate_violin_matches_host_restatement():
    from hero_b200 import evalpass
    g = torch.Generator().manual_seed(0)
    scores = [torch.randn(4, 1, generator=g) * 3, torch.randn(2, 1, generator=g) * 3]
    scores[0][1, 0] = 0.0                      # sigmoid(0) = 0.5 is not > 0.5: predicted 0
    targets = [torch.tensor([[1], [0], [0], [1]]), torch.tensor([[1], [1]])]
    qids = [[10, 11, 12, 13], [14, 15]]
    loader = [{"qids": list(q), "targets": t} for q, t in zip(qids, targets)]
    val_log, results, logits = evalpass.validate_violin(_Fixed(scores), loader, "test",
                                                        save_logits=True)
    loss, acc, ref_results, ref_logits = _host_validate_violin(zip(qids, scores, targets), True)
    assert set(val_log) == {"valid/test_loss", "valid/test_acc", "valid/test_ex_per_s"}
    assert val_log["valid/test_loss"] == pytest.approx(loss, rel=1e-6)
    assert val_log["valid/test_acc"] == acc
    assert val_log["valid/test_ex_per_s"] > 0
    assert results == ref_results and results["11"] == 0
    assert logits == ref_logits
    assert all(isinstance(v, list) and len(v) == 1 for v in logits.values())
    # without save_logits no logits are kept
    loader = [{"qids": list(q), "targets": t} for q, t in zip(qids, targets)]
    _, results2, logits2 = evalpass.validate_violin(_Fixed(scores), loader, "val")
    assert results2 == ref_results and logits2 == {}


def test_validate_violin_takes_a_one_row_batch():
    """A one-row batch (the last batch of a split can be one) works; its numbers are those of the
    same row evaluated in a larger batch."""
    from hero_b200 import evalpass
    scores = [torch.tensor([[2.0], [-1.0]]), torch.tensor([[-0.5]])]
    targets = [torch.tensor([[1], [1]]), torch.tensor([[0]])]
    loader = [{"qids": [1, 2], "targets": targets[0]}, {"qids": [3], "targets": targets[1]}]
    val_log, results, logits = evalpass.validate_violin(_Fixed(scores), loader, "val",
                                                        save_logits=True)
    merged = [([1, 2, 3], torch.cat(scores), torch.cat(targets))]
    loss, acc, ref_results, ref_logits = _host_validate_violin(merged, True)
    assert val_log["valid/val_loss"] == pytest.approx(loss, rel=1e-6)
    assert val_log["valid/val_acc"] == acc == 2 / 3
    assert results == ref_results == {"1": 1, "2": 0, "3": 0}
    assert logits == ref_logits
