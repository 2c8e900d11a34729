"""TEST INFRASTRUCTURE: torch restatements of the pretraining-validation entry points
(include/hero_b200.h: hero_ce_finish_stats behind ops.lm_head_ce_stats, and hero_row_l2_cos), in
the style of tests/fake_ops.py, so evalpass.validate_pretrain runs on a CPU-only box. The hit is
`label logit >= row max` (an exact tie counts), cosine is torch's F.cosine_similarity."""
import torch
import torch.nn.functional as F

from tests import fake_ops


def _add(acc, a, b):
    if acc is not None:
        acc += torch.stack([a.sum(), b.sum().float()])


def lm_head_ce_stats(h, emb, bias, labels, n_valid, acc=None):
    logits = h.float() @ emb.float().t()
    if bias is not None:
        logits = logits + bias
    logits = logits[:, :n_valid]
    lse = torch.logsumexp(logits, dim=-1)
    lab = logits.gather(1, labels.long()[:, None])[:, 0]
    loss = lse - lab
    hit = (lab >= logits.max(dim=-1).values).to(torch.int32)
    _add(acc, loss, hit)
    return loss, lse, hit


def row_l2_cos(x, y, acc=None, eps=1e-8):
    from hero_b200 import ops
    ops._row_stats_bounds("row_l2_cos", x.shape[0], x.shape[1])
    l2 = (x.float() - y.float()).pow(2).sum(dim=1).sqrt()
    cos = F.cosine_similarity(x.float(), y.float(), dim=-1, eps=eps)
    _add(acc, l2, cos)
    return l2, cos


def install(monkeypatch):
    fake_ops.install(monkeypatch)
    from hero_b200 import ops
    monkeypatch.setattr(ops, "lm_head_ce_stats", lm_head_ce_stats)
    monkeypatch.setattr(ops, "row_l2_cos", row_l2_cos)
