"""The segment-table optimizer kernels on the H100 (csrc/optim.cu: hero_adamw_step_groups,
hero_sumsq_segments_f32): bitwise equality with the single-range kernel run per segment, gaps left
untouched, the sum of squares against float64, argument checks, one launch per step, a training
step of HeroForVideoQA with lr_mul = 10 without host synchronisation, and three steps against the
reference's own AdamW and build_optimizer staged under oracle/_ref."""
import types

import pytest
import torch

from tests import test_videoqa_cpu as qa_cpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SENTINEL = 12345.0


def _table(seed, n_groups=None):
    """Random segments: lengths multiples of 4 but not of 64, some adjacent, some with gaps."""
    g = torch.Generator().manual_seed(seed)
    n_groups = n_groups or int(torch.randint(1, 9, (1,), generator=g))
    segs, pos = [], 0
    for _ in range(int(torch.randint(1, 40, (1,), generator=g))):
        if float(torch.rand(1, generator=g)) < 0.5:
            pos += 4 * int(torch.randint(1, 50, (1,), generator=g))     # gap
        length = 4 * int(torch.randint(1, 4000, (1,), generator=g))
        if length % 64 == 0:
            length += 4
        segs.append((pos, length, int(torch.randint(0, n_groups, (1,), generator=g))))
        pos += length
    return segs, pos + 4 * int(torch.randint(0, 20, (1,), generator=g)), n_groups


def _buffers(n, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g)
    grad = torch.randn(n, generator=g) * 0.1
    m = torch.randn(n, generator=g) * 0.01
    v = torch.rand(n, generator=g) * 1e-3
    return [t.to(DEV) for t in (p, grad, m, v)] + [p.to(DEV).to(torch.bfloat16)]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("clip", [False, True])
def test_grouped_step_is_bitwise_the_per_segment_kernel(seed, clip):
    from hero_b200 import ops
    segs, n, n_groups = _table(seed)
    table = ops.SegmentTable(segs, n, n_groups, DEV)
    g = torch.Generator().manual_seed(100 + seed)
    lrs = (torch.rand(n_groups, generator=g) * 1e-3).tolist()
    wds = [0.0 if k % 2 else 0.01 for k in range(n_groups)]
    step_sizes = [lr * 0.7 for lr in lrs]
    lr_wds = [lr * wd for lr, wd in zip(lrs, wds)]
    p, grad, m, v, mirror = _buffers(n, seed)
    inside = torch.zeros(n, dtype=torch.bool, device=DEV)
    for a, length, _ in segs:
        inside[a:a + length] = True
    for t in (p, m, v, mirror):
        t[~inside] = SENTINEL
    sumsq = torch.full((1,), 40.0, device=DEV) if clip else None
    kw = dict(beta1=0.9, beta2=0.98, eps=1e-6, grad_scale=0.5, clip_sumsq=sumsq,
              clip_max_norm=3.0 if clip else 0.0)
    a_bufs = [t.clone() for t in (p, m, v, mirror)]
    ops.adamw_step_groups(a_bufs[0], grad, a_bufs[1], a_bufs[2], a_bufs[3], table,
                          step_sizes=step_sizes, lr_wds=lr_wds, **kw)
    b_bufs = [t.clone() for t in (p, m, v, mirror)]
    for a, length, grp in segs:
        sl = slice(a, a + length)
        ops.adamw_step(b_bufs[0][sl], grad[sl], b_bufs[1][sl], b_bufs[2][sl], b_bufs[3][sl],
                       step_size=step_sizes[grp], lr_wd=lr_wds[grp], **kw)
    torch.cuda.synchronize()
    for name, x, y, orig in zip(("p", "m", "v", "bf16"), a_bufs, b_bufs, (p, m, v, mirror)):
        assert torch.equal(x, y), name
        assert torch.equal(x[~inside], orig[~inside]), name           # gaps untouched
        assert not torch.equal(x[inside], orig[inside]), name


@pytest.mark.parametrize("seed", range(4))
def test_sumsq_segments_matches_float64(seed):
    from hero_b200 import ops
    segs, n, n_groups = _table(50 + seed)
    table = ops.SegmentTable(segs, n, n_groups, DEV)
    x = torch.randn(n, generator=torch.Generator().manual_seed(seed)).to(DEV)
    out = torch.full((1,), 0.25, device=DEV)
    ops.sumsq_segments(x, table, out)
    ref = 0.25 + sum(float((x[a:a + length].double() ** 2).sum()) for a, length, _ in segs)
    assert abs(float(out) - ref) <= 1e-5 * ref


def test_bad_arguments_raise_before_any_launch():
    from hero_b200 import _lib, ops
    n = 256
    p, grad, m, v, mirror = _buffers(n, 0)
    with pytest.raises(ValueError, match="groups"):
        ops.SegmentTable([(0, 64, 0)], n, 9, DEV)
    with pytest.raises(ValueError, match="not inside"):
        ops.SegmentTable([(240, 64, 0)], n, 1, DEV)
    with pytest.raises(ValueError, match="group 3"):
        ops.SegmentTable([(0, 64, 3)], n, 2, DEV)
    with pytest.raises(ValueError, match="overlaps"):
        ops.SegmentTable([(0, 64, 0), (32, 64, 1)], n, 2, DEV)
    table = ops.SegmentTable([(0, 64, 0)], n, 1, DEV)
    with pytest.raises(ValueError, match="describes"):
        ops.sumsq_segments(p[:128], table, torch.zeros(1, device=DEV))
    # the library's own checks (on the host copy of the table), behind the Python ones
    before = [t.clone() for t in (p, m, v, mirror)]
    kw = dict(step_sizes=[1e-3], lr_wds=[0.0], beta1=0.9, beta2=0.98, eps=1e-6)
    bad = ops.SegmentTable([(0, 64, 0)], n, 1, DEV)
    bad.host[0, 0] = 224                                  # [224, 288) runs past n
    with pytest.raises(_lib.HeroError, match="not inside"):
        ops.adamw_step_groups(p, grad, m, v, mirror, bad, **kw)
    bad = ops.SegmentTable([(0, 64, 0)], n, 1, DEV)
    bad.host[0, 2] = 1
    with pytest.raises(_lib.HeroError, match="group 1"):
        ops.adamw_step_groups(p, grad, m, v, mirror, bad, **kw)
    bad = ops.SegmentTable([(0, 64, 0)], n, 1, DEV)
    bad.n_groups = 9
    with pytest.raises(_lib.HeroError, match="9 groups"):
        ops.sumsq_segments(p, bad, torch.zeros(1, device=DEV))
    torch.cuda.synchronize()
    for x, y in zip((p, m, v, mirror), before):
        assert torch.equal(x, y)


def _opts(lr_mul=10.0):
    return types.SimpleNamespace(optim="adamw", learning_rate=5e-5, lr_mul=lr_mul,
                                 betas=[0.9, 0.98], weight_decay=0.01, grad_norm=1.0)


def _tiny_step(tmp_path, lr_mul=10.0, freeze=False):
    from hero_b200 import synth
    from hero_b200.optim import build_optimizer
    from hero_b200.plan import attach_plan
    vx = qa_cpu.fixture()
    model = qa_cpu.qa_model(tmp_path, vx).to(DEV).train()
    if freeze:
        model.v_encoder.f_encoder.embeddings.word_embeddings.weight.requires_grad_(False)
    opt = build_optimizer(model, _opts(lr_mul))
    batch = synth.to_device(attach_plan(qa_cpu.qa_batch(vx), kind="videoqa"), DEV)
    return model, opt, batch


@pytest.mark.parametrize("freeze", [False, True])
def test_one_launch_per_step(tmp_path, freeze):
    from hero_b200 import ops
    _, opt, _ = _tiny_step(tmp_path, freeze=freeze)
    assert len(opt.param_groups) == 4 and opt._partial == freeze
    ops.reset_launch_count()
    opt.step()
    assert ops.launch_count() == 1
    opt.clip_grad_norm_device_(1.0)
    opt.step()
    assert ops.launch_count() == 3


def test_training_step_with_lr_mul_does_not_sync(tmp_path):
    model, opt, batch = _tiny_step(tmp_path)
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.zero_grad()
        qa_loss, t_loss = model(batch, "tvqa")
        (qa_loss + 0.4 * t_loss).backward()
        for i, group in enumerate(opt.param_groups):
            group["lr"] = 3e-5 * (10.0 if i < 2 else 1.0)
        opt.clip_grad_norm_device_(1.0)
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(qa_loss) and torch.isfinite(t_loss)
    moved = [n for n, p in model.named_parameters() if not torch.equal(p.detach(), before[n])]
    assert "qa_pred_head.linear_1.weight" in moved
    assert "v_encoder.c_encoder.encoder.layer.0.output.dense.weight" in moved


def test_three_steps_match_the_reference_adamw():
    """Gradients of one real HeroForVideoQA step (6 + 3 layers, H 768) copied into the reference
    model; three steps of the reference's AdamW from its own build_optimizer and three of ours,
    with the train_videoQA.py:186-192 schedule at lr_mul = 10, agree within 1e-6 relative."""
    from tests.test_videoqa_gpu import _reference_module, _tvqa_model
    VideoModelConfig, RefQA = _reference_module()
    from optim.misc import build_optimizer as ref_build_optimizer
    from hero_b200 import synth
    from hero_b200.optim import build_optimizer
    model, path = _tvqa_model(seed=4)
    ref = RefQA(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(model.state_dict())
    model, ref = model.to(DEV).train(), ref.to(DEV)
    o = _opts()
    opt = build_optimizer(model, o)
    ref_opt = ref_build_optimizer(ref, o)
    qa_loss, t_loss = model(synth.to_device(synth.syn_tvqa(seed=9), DEV), "tvqa")
    (qa_loss + 0.4 * t_loss).backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()}
    for n, p in ref.named_parameters():
        p.grad = grads[n].clone()
    for lr_this_step in (2e-5, 5e-5, 3e-5):
        for optimizer in (opt, ref_opt):
            for i, param_group in enumerate(optimizer.param_groups):
                if i == 0 or i == 1:
                    param_group['lr'] = lr_this_step * o.lr_mul
                elif i == 2 or i == 3:
                    param_group['lr'] = lr_this_step
                else:
                    raise ValueError()
        opt.step()
        ref_opt.step()
    ours = dict(model.named_parameters())
    worst = max(float((ours[n].detach() - p.detach()).norm() / p.detach().norm().clamp(min=1e-30))
                for n, p in ref.named_parameters())
    print(f"max relative parameter difference after three steps: {worst:.3e}")
    assert worst < 1e-6
