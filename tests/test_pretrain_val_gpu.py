"""Pretraining validation on the GPU: hero_ce_finish_stats and hero_row_l2_cos (csrc/optim.cu)
against hero_ce_finish / torch, and evalpass.validate_pretrain against the reference's fixture
(tests/test_pretrain_val_cpu.py) with one device->host copy per task."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ce_operands(n, V, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = (torch.randn(n, K, generator=g, device=DEV) * 0.5).to(torch.bfloat16)
    emb = (torch.randn(V, K, generator=g, device=DEV) * 0.5).to(torch.bfloat16)
    bias = torch.randn(V, generator=g, device=DEV) * 0.1
    labels = torch.randint(0, V - 24, (n,), generator=g, device=DEV, dtype=torch.int32)
    return h, emb, bias, labels


@pytest.mark.parametrize("n, V, K", [(1, 64, 64), (300, 1024, 768), (1000, 50272, 768)])
def test_ce_finish_stats_matches_ce_finish_and_argmax(n, V, K):
    from hero_b200 import ops
    h, emb, bias, labels = _ce_operands(n, V, K, seed=n)
    n_valid = V - 16
    logits = (h.float() @ emb.float().t() + bias)[:, :n_valid]
    # half the rows labelled with their fp32 argmax: hits, across many 64-column slabs
    half = torch.arange(n, device=DEV) % 2 == 0
    labels = torch.where(half, logits.argmax(dim=-1).int(), labels)
    partial, lab = ops.lm_head_ce_partials(h, emb, bias, labels, n_valid)
    loss0, lse0 = ops.ce_finish(partial, lab)
    acc1 = torch.zeros(2, device=DEV)
    acc2 = torch.zeros(2, device=DEV)
    loss, lse, hit = ops.ce_finish_stats(partial, lab, acc=acc1)
    ops.ce_finish_stats(partial, lab, acc=acc2)
    torch.cuda.synchronize()
    assert torch.equal(loss.view(torch.int32), loss0.view(torch.int32))
    assert torch.equal(lse.view(torch.int32), lse0.view(torch.int32))
    assert torch.equal(acc1.view(torch.int32), acc2.view(torch.int32))     # fixed order
    assert float(acc1[1]) == float(hit.sum())
    assert abs(float(acc1[0]) - float(loss.double().sum())) <= 1e-5 * float(loss.abs().sum())
    top2 = logits.topk(2, dim=-1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-3
    want = logits.argmax(dim=-1) == labels.long()
    assert torch.equal(hit.bool()[clear], want[clear])
    assert int(hit[clear].sum()) >= int(clear[half].sum())     # the argmax-labelled rows hit
    if V > 64:
        assert len(set((labels[half].long() // 64).tolist())) > 1 or n == 1
    # the fused pair gives the same
    l2, _, h2 = ops.lm_head_ce_stats(h, emb, bias, labels, n_valid)
    assert torch.equal(l2.view(torch.int32), loss0.view(torch.int32)) and torch.equal(h2, hit)


def test_exact_tie_counts_as_hit():
    """Stated deviation: on an exact tie the label counts as a hit, where torch.max (the
    reference) reports the lower tied index."""
    from hero_b200 import ops
    h, emb, bias, labels = _ce_operands(4, 128, 64, seed=5)
    emb[2] = h[0] * 4
    emb[5] = h[0] * 4                   # columns 2 and 5 of row 0: equal, and the row maximum
    labels[0] = 5
    bias.zero_()
    partial, lab5 = ops.lm_head_ce_partials(h, emb, bias, labels, 128)
    _, _, hit = ops.ce_finish_stats(partial, lab5)
    labels2 = labels.clone()
    labels2[0] = 2
    _, lab2 = ops.lm_head_ce_partials(h, emb, bias, labels2, 128)
    # the GEMM's own values: columns 2 and 5 equal, and the row maximum (max over the slabs)
    row_max = float(partial[:, 0, 0].max())
    assert float(lab5[0]) == float(lab2[0]) == row_max
    logits = h.float() @ emb.float().t()
    assert int(logits[0].argmax()) == 2             # torch.max reports the lower tied index
    assert int(hit[0]) == 1


@pytest.mark.parametrize("m, d", [(37, 64), (300, 4352), (5, 63), (1, 4352)])
def test_row_l2_cos_matches_fp64(m, d):
    from hero_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(m + d)
    x = torch.randn(m, d, generator=g, device=DEV)
    y = x + 0.7 * torch.randn(m, d, generator=g, device=DEV)
    x[m // 2] = 0.0                     # a zero row: cosine 0 (norm clamped at eps)
    acc1 = torch.zeros(2, device=DEV)
    acc2 = torch.zeros(2, device=DEV)
    l2, cos = ops.row_l2_cos(x, y, acc=acc1)
    ops.row_l2_cos(x, y, acc=acc2)
    torch.cuda.synchronize()
    xd, yd = x.double(), y.double()
    l2_ref = (xd - yd).pow(2).sum(1).sqrt()
    cos_ref = torch.nn.functional.cosine_similarity(xd, yd, dim=-1, eps=1e-8)
    assert float(((l2.double() - l2_ref).abs() / l2_ref).max()) < 1e-5
    assert float((cos.double() - cos_ref).abs().max()) < 1e-5
    assert float(cos[m // 2]) == 0.0
    assert torch.equal(acc1.view(torch.int32), acc2.view(torch.int32))
    assert abs(float(acc1[0]) - float(l2_ref.sum())) <= 1e-5 * float(l2_ref.sum())
    assert abs(float(acc1[1]) - float(cos_ref.sum())) <= 1e-5 * m


@pytest.mark.parametrize("m, d", [(4, 0), (4, 4353), (4, 8192), ((1 << 24) + 1, 1)])
def test_row_l2_cos_out_of_bounds_raise_before_launch(m, d):
    from hero_b200 import ops
    x = torch.randn(m, max(d, 1), device=DEV)[:, :d]
    acc = torch.full((2,), float("nan"), device=DEV)
    with pytest.raises(ValueError):
        ops.row_l2_cos(x, x.clone(), acc=acc)
    torch.cuda.synchronize()
    assert bool(torch.isnan(acc).all())            # nothing ran


def test_ce_finish_stats_out_of_bounds_raise_before_launch():
    from hero_b200 import ops
    m = (1 << 24) + 1
    partial = torch.zeros((1, m, 2), device=DEV)
    lab = torch.zeros(m, device=DEV)
    acc = torch.full((2,), float("nan"), device=DEV)
    with pytest.raises(ValueError):
        ops.ce_finish_stats(partial, lab, acc=acc)
    torch.cuda.synchronize()
    assert bool(torch.isnan(acc).all())


@pytest.mark.parametrize("attach", [False, True])
def test_validate_pretrain_matches_reference_on_device(tmp_path, attach):
    from hero_b200 import ops
    from tests.test_pretrain_val_cpu import run_fixture_comparison
    run_fixture_comparison(tmp_path, ops, DEV, attach=attach)


def test_fused_mlm_and_nce_at_real_dimensions_against_fp32_logits():
    """validate_mlm / validate_mfm_nce at real dimensions (6 + 3 layers, H 768, vocabulary
    50 272, 4352-d features; SYN-HT100M-dense batches) against the model's own fp32 torch logits
    (head.decoder, mfm_nce): the loss error of the fused bf16-operand GEMM is at most 1.5x that of
    the same logits under bf16 autocast (SURVEY §8c), and hits agree away from near-ties."""
    from hero_b200 import evalpass, synth
    from tests import pretrain_val_batches as pv
    model = pv.real_model(DEV)
    for task, fn in (("mlm", evalpass.validate_mlm), ("mfm-nce", evalpass.validate_mfm_nce)):
        batches = [synth.to_device(pv.real_batch(task, i), DEV) for i in range(2)]
        l32, h32, n, gap = pv.torch_logit_metrics(model, task, batches)
        lac, _, _, _ = pv.torch_logit_metrics(model, task, batches, autocast=True)
        got = fn(model, batches)
        err, yard = abs(got["loss"] - l32 / n), abs(lac - l32) / n
        print(f"{task}: rows {n}, fp32 loss {l32 / n:.6f}, fused err {err:.3e}, "
              f"autocast err {yard:.3e}")
        assert err <= 1.5 * yard + 1e-6 * abs(l32 / n), (task, err, yard)
        near = int((gap <= 2e-2).sum())
        assert abs(round(got["acc"] * n) - h32) <= near, (task, got["acc"] * n, h32, near)


def test_validate_pretrain_one_copy_per_task(tmp_path):
    from hero_b200 import evalpass
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model, loaders
    model = build_model(tmp_path, gu.load("pretrain_val_tiny.npz"), DEV)
    ld = loaders(DEV, attach=True)
    evalpass.validate_pretrain(model, ld, pv.Opts)           # warm-up (library load, caches)
    ld = loaders(DEV, attach=True)
    torch.cuda.synchronize()
    copies = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(t, *a, **k):
        if t.is_cuda:
            copies.append(tuple(t.shape))
        return real_cpu(t, *a, **k)

    try:
        torch.Tensor.cpu = counting_cpu
        out = evalpass.validate_pretrain(model, ld, pv.Opts)
    finally:
        torch.Tensor.cpu = real_cpu
    assert len(copies) == len(pv.TASKS), copies
    assert all(np.isfinite(v) for v in out.values())
    assert model.training
