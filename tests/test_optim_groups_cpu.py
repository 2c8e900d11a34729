"""FusedAdamW with the reference's four parameter groups (optim/misc.py:14-50) on the host, with
hero_b200.ops routed through tests/fake_optim_groups_ops.py: group membership against the
reference's own build_optimizer, the update of the fine-tuning loops (lr_mul, train_videoQA.py:
186-192) against the reference rule, frozen parameters, and the state round trip. The CUDA
kernels are covered by test_optim_groups_gpu.py."""
import json
import types

import pytest
import torch

from oracle import hero_oracle as orc
from tests import fake_optim_groups_ops
from tests import test_tvc_cpu as tvc
from tests import test_videoqa_cpu as qa
from tests import test_violin_cpu as violin

LR, WD, BETAS = 5e-5, 0.01, (0.9, 0.98)


def opts(lr_mul=10.0):
    """The optimizer fields of config/train-tvqa-8gpu.json."""
    return types.SimpleNamespace(optim="adamw", learning_rate=LR, lr_mul=lr_mul, betas=list(BETAS),
                                 weight_decay=WD, grad_norm=1.0)


def group_of(name, lr, lr_mul):
    """(lr, weight_decay) of a parameter under optim/misc.py:14-50 and train_videoQA.py:186-192."""
    lr = lr if "v_encoder" in name else lr * lr_mul
    return lr, 0.0 if any(nd in name for nd in ("bias", "LayerNorm.bias", "LayerNorm.weight")) else WD


def group_names(model, opt):
    """Names of the parameters inside each group's flat ranges."""
    off = {id(p): o for _, p, o, _ in opt.flat.entries}
    out = []
    for g in opt.param_groups:
        out.append(sorted(n for n, p in model.named_parameters()
                          if any(a <= off[id(p)] < b for a, b in g["ranges"])))
    return out


def videoqa_model(tmp_path):
    return qa.qa_model(tmp_path, qa.fixture())


def _reference():
    from oracle import gen_golden as gg
    from oracle import stage_ref
    ref = stage_ref.available()
    if ref is None:
        pytest.skip("no staged reference under oracle/_ref")
    gg.REF = ref
    gg.install_stubs()


def _reference_model(kind, tmp_path):
    """(our tiny model, the reference's model class on the same configuration)."""
    _reference()
    from model.model import VideoModelConfig
    if kind == "videoqa":
        from model.videoQA import HeroForVideoQA
        ours = qa.qa_model(tmp_path, qa.fixture())
        c = json.loads(str(qa.fixture()["config"]))
        ref = HeroForVideoQA(VideoModelConfig(str(tmp_path / "qa.json")), c["vfeat_dim"],
                             c["max_frm_seq_len"])
    elif kind == "violin":
        from model.violin import HeroForViolin
        ours = violin.violin_model(tmp_path, violin.fixture())
        c = json.loads(str(violin.fixture()["config"]))
        ref = HeroForViolin(VideoModelConfig(str(tmp_path / "violin.json")), c["vfeat_dim"],
                            c["max_frm_seq_len"])
    else:
        from model.tvc import HeroForTvc
        ours = tvc.tvc_model(tmp_path, tvc.fixture())
        c = json.loads(str(tvc.fixture()["config"]))
        ref = HeroForTvc(VideoModelConfig(str(tmp_path / "tvc.json")), c["vfeat_dim"],
                         c["max_frm_seq_len"], lsr=0.1)
    return ours, ref


@pytest.mark.parametrize("kind", ["videoqa", "violin", "tvc"])
def test_groups_match_the_reference_build_optimizer(tmp_path, monkeypatch, kind):
    fake_optim_groups_ops.install(monkeypatch)
    from hero_b200.optim import build_optimizer
    ours, ref = _reference_model(kind, tmp_path)
    from optim.misc import build_optimizer as ref_build_optimizer
    o = opts()
    opt = build_optimizer(ours, o, device=torch.device("cpu"))
    ref_opt = ref_build_optimizer(ref, o)
    ref_names = {id(p): n for n, p in ref.named_parameters()}
    assert len(opt.param_groups) == len(ref_opt.param_groups) == 4
    for ours_names, g, rg in zip(group_names(ours, opt), opt.param_groups, ref_opt.param_groups):
        assert ours_names == sorted(ref_names[id(p)] for p in rg["params"])
        assert g["lr"] == rg["lr"] and g["weight_decay"] == rg["weight_decay"]
    assert sum(map(len, group_names(ours, opt))) == len(list(ours.parameters()))


def _random_grads(model, gen):
    grads = {n: torch.randn(p.shape, generator=gen) * 0.1 for n, p in model.named_parameters()}
    for n, p in model.named_parameters():
        p.grad.copy_(grads[n])
    return grads


def test_update_matches_the_reference_rule_with_lr_mul(tmp_path, monkeypatch):
    """Three steps of the train_videoQA.py:186-192 loop (lr_mul = 10) with global-norm clipping:
    every parameter follows optim/adamw.py:80-104 with its group's lr and weight decay."""
    fake_optim_groups_ops.install(monkeypatch)
    from hero_b200.optim import build_optimizer
    model = videoqa_model(tmp_path)
    o = opts()
    optimizer = build_optimizer(model, o, device=torch.device("cpu"))
    assert len(optimizer.param_groups) == 4
    ref = {n: [p.detach().clone(), torch.zeros_like(p), torch.zeros_like(p)]
           for n, p in model.named_parameters()}
    gen = torch.Generator().manual_seed(5)
    for global_step, lr_this_step in enumerate([2e-5, 5e-5, 3e-5], start=1):
        optimizer.zero_grad()
        grads = _random_grads(model, gen)
        # learning rate scheduling (train_videoQA.py:186-192, verbatim)
        for i, param_group in enumerate(optimizer.param_groups):
            if i == 0 or i == 1:
                param_group['lr'] = lr_this_step * o.lr_mul
            elif i == 2 or i == 3:
                param_group['lr'] = lr_this_step
            else:
                raise ValueError()
        total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
        assert abs(optimizer.clip_grad_norm_(o.grad_norm) - total) < 1e-5 * total
        scale = min(1.0, o.grad_norm / (total + 1e-6))
        optimizer.step()
        for n, (p, m, v) in ref.items():
            lr, wd = group_of(n, lr_this_step, o.lr_mul)
            ref[n] = list(orc.adamw_step(p, grads[n] * scale, m, v, global_step, lr, *BETAS, 1e-6,
                                         wd))
        for n, p in model.named_parameters():
            assert (p.detach() - ref[n][0]).abs().max() < 2e-6, (n, global_step)


def test_frozen_parameters_are_left_alone(tmp_path, monkeypatch):
    """Frozen word embeddings and one encoder layer: bitwise unchanged (masters, bf16 mirror),
    moments zero, and the clip norm counts only the trainable gradients."""
    fake_optim_groups_ops.install(monkeypatch)
    from hero_b200.optim import build_optimizer
    model = videoqa_model(tmp_path)
    frozen = [n for n, p in model.named_parameters()
              if n == "v_encoder.f_encoder.embeddings.word_embeddings.weight"
              or n.startswith("v_encoder.f_encoder.encoder.layer.0.")]
    assert len(frozen) > 10
    for n, p in model.named_parameters():
        p.requires_grad_(n not in frozen)
    o = opts(lr_mul=1.0)
    opt = build_optimizer(model, o, device=torch.device("cpu"))
    assert len(opt.param_groups) == 4 and opt._partial
    params = dict(model.named_parameters())
    before = {n: p.detach().clone() for n, p in params.items()}
    mirror = {n: opt.flat.bf16(params[n]).clone() for n in frozen}
    gen = torch.Generator().manual_seed(6)
    for _ in range(2):
        opt.zero_grad()
        grads = _random_grads(model, gen)
        total = torch.sqrt(sum((g.double() ** 2).sum() for n, g in grads.items()
                               if n not in frozen)).item()
        assert abs(opt.clip_grad_norm_(o.grad_norm) - total) < 1e-5 * total
        opt.step()
    off = {n: (o_, k) for n, _, o_, k in opt.flat.entries}
    for n in frozen:
        assert torch.equal(params[n].detach(), before[n]), n
        assert torch.equal(opt.flat.bf16(params[n]), mirror[n]), n
        a, k = off[n]
        assert not opt.exp_avg[a:a + k].any() and not opt.exp_avg_sq[a:a + k].any(), n
    for n in params:
        if n not in frozen:
            assert not torch.equal(params[n].detach(), before[n]), n


def test_four_group_state_round_trip(tmp_path, monkeypatch):
    fake_optim_groups_ops.install(monkeypatch)
    from hero_b200.optim import build_optimizer
    o = opts()

    def make(sub):
        d = tmp_path / sub
        d.mkdir()
        m = videoqa_model(d)
        return m, build_optimizer(m, o, device=torch.device("cpu"))

    def step(m, opt, grads, lr):
        opt.zero_grad()
        for n, p in m.named_parameters():
            p.grad.copy_(grads[n])
        for i, g in enumerate(opt.param_groups):
            g["lr"] = lr * (o.lr_mul if i < 2 else 1.0)
        opt.clip_grad_norm_(o.grad_norm)
        opt.step()

    m1, opt1 = make("a")
    gen = torch.Generator().manual_seed(7)
    all_grads = [{n: torch.randn(p.shape, generator=gen) * 0.1 for n, p in m1.named_parameters()}
                 for _ in range(3)]
    step(m1, opt1, all_grads[0], 2e-5)
    step(m1, opt1, all_grads[1], 4e-5)
    sd = {k: v.clone() if torch.is_tensor(v) else v for k, v in opt1.state_dict().items()}
    assert [(g["lr"], g["weight_decay"]) for g in sd["param_groups"]] == \
        [(4e-5 * o.lr_mul, WD), (4e-5 * o.lr_mul, 0.0), (4e-5, WD), (4e-5, 0.0)]
    weights = {k: v.clone() for k, v in m1.state_dict().items()}
    step(m1, opt1, all_grads[2], 3e-5)

    m2, opt2 = make("b")
    m2.load_state_dict(weights)
    opt2.load_state_dict(sd)
    assert opt2.step_count == 2
    assert [g["lr"] for g in opt2.param_groups] == [g["lr"] for g in sd["param_groups"]]
    step(m2, opt2, all_grads[2], 3e-5)
    for (n, a), (_, b) in zip(m2.named_parameters(), m1.named_parameters()):
        assert torch.equal(a.detach(), b.detach()), n

    two = build_optimizer(videoqa_model(tmp_path), opts(lr_mul=1.0), device=torch.device("cpu"))
    assert len(two.param_groups) == 2
    with pytest.raises(ValueError, match="parameter groups"):
        opt2.load_state_dict(two.state_dict())


def test_lr_mul_one_keeps_two_groups(tmp_path, monkeypatch):
    fake_optim_groups_ops.install(monkeypatch)
    from hero_b200.optim import build_optimizer
    opt = build_optimizer(videoqa_model(tmp_path), opts(lr_mul=1.0), device=torch.device("cpu"))
    assert len(opt.param_groups) == 2 and opt._segments is None
    assert [g["range"] for g in opt.param_groups] == [(0, opt.flat.no_decay_start),
                                                       (opt.flat.no_decay_start, opt.flat.total)]


def test_other_optimizers_stay_refused(tmp_path, monkeypatch):
    fake_optim_groups_ops.install(monkeypatch)
    from hero_b200.optim import build_optimizer
    for name in ("adam", "adamax"):
        o = opts()
        o.optim = name
        with pytest.raises(ValueError, match="adamw"):
            build_optimizer(videoqa_model(tmp_path), o, device=torch.device("cpu"))


@pytest.mark.parametrize("segments,n_groups,match", [
    ([(0, 8, 0)], 9, "groups"),
    ([(0, 8, 0)], 0, "groups"),
    ([(0, 8, 2)], 2, "group 2"),
    ([(0, 8, -1)], 2, "group -1"),
    ([(60, 8, 0)], 1, "not inside"),
    ([(-4, 8, 0)], 1, "not inside"),
    ([(2, 8, 0)], 1, "multiples of 4"),
    ([(0, 6, 0)], 1, "multiples of 4"),
    ([(0, 16, 0), (8, 8, 1)], 2, "overlaps"),
])
def test_segment_table_rejects_bad_tables(segments, n_groups, match):
    from hero_b200 import ops
    with pytest.raises(ValueError, match=match):
        ops.SegmentTable(segments, 64, n_groups, torch.device("cpu"))
    table = ops.SegmentTable([(32, 16, 1), (0, 8, 0), (48, 16, 0)], 64, 2, torch.device("cpu"))
    assert table.host.tolist() == [[0, 8, 0], [32, 16, 1], [48, 16, 0]] and table.covered == 40
