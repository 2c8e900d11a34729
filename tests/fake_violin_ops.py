"""TEST INFRASTRUCTURE: torch restatement of the single-pooling mode of the video QA pooling entry
points (include/hero_b200.h: hero_qa_pool_fwd / hero_qa_pool_bwd with w_st == NULL), so
HeroForViolin runs on a CPU-only box. The expressions are those of model/violin.py:30-47 on the
(Nv*Nq, L, H) tensor gathered through the frame map (zeros where it is -1). Two-pooling calls go
to tests/fake_qa_ops.py. Also used on the GPU as the fp32 restatement the kernels are checked
against."""
import torch

from tests import fake_qa_ops


def pool_ref(x, mask, w):
    """model/violin.py:30-47 on x (N, L, H), mask (N, L): (pooled (N, H), a (N*L))."""
    m = mask.unsqueeze(-1)
    a = torch.softmax((x @ w.reshape(-1, 1)) * m + (1 - m) * -1e4, dim=1)
    pooled = torch.einsum("vlm,vld->vmd", a, x).squeeze(1)
    return pooled, a.reshape(-1)


def _rows(h, frame_map, nv, nq, length):
    return fake_qa_ops.padded(h, frame_map, nv * nq, 1, length).view(nv * nq, length, h.shape[1])


def qa_pool_fwd(h, frame_map, mask, w_qa, w_st, nv, nq, length, a, b, qa_pooled, st_pooled):
    if w_st is not None:
        return fake_qa_ops.qa_pool_fwd(h, frame_map, mask, w_qa, w_st, nv, nq, length, a, b,
                                       qa_pooled, st_pooled)
    from hero_b200 import _lib, ops
    ops._qa_bounds(nv, nq, length, h.shape[1])
    if b is not None or st_pooled is not None:
        raise _lib.HeroError("qa_pool_fwd: w_st, b and st_pooled must be all set or all NULL")
    pooled, pa = pool_ref(_rows(h, frame_map, nv, nq, length), mask.view(nv * nq, length), w_qa)
    a.copy_(pa)
    qa_pooled.copy_(pooled)


def qa_pool_bwd(h, frame_map, mask, w_qa, w_st, a, b, d_qa, d_st, nv, nq, length, dh, dw_qa,
                dw_st):
    if w_st is not None:
        return fake_qa_ops.qa_pool_bwd(h, frame_map, mask, w_qa, w_st, a, b, d_qa, d_st, nv, nq,
                                       length, dh, dw_qa, dw_st)
    from hero_b200 import _lib, ops
    ops._qa_bounds(nv, nq, length, h.shape[1])
    if b is not None or d_st is not None or dw_st is not None:
        raise _lib.HeroError("qa_pool_bwd: w_st, b, d_st_pooled and dw_st must be all set or all "
                             "NULL")
    with torch.enable_grad():
        x = _rows(h, frame_map, nv, nq, length).detach().requires_grad_(True)
        w = w_qa.detach().clone().requires_grad_(True)
        pooled, _ = pool_ref(x, mask.view(nv * nq, length), w)
        pooled.backward(d_qa)
    m = frame_map.long()
    keep = m >= 0
    dh[m[keep]] = x.grad.reshape(-1, h.shape[1])[keep]
    dw_qa.add_(w.grad)


def install(monkeypatch):
    fake_qa_ops.install(monkeypatch)
    from hero_b200 import ops
    for name in ("qa_pool_fwd", "qa_pool_bwd"):
        monkeypatch.setattr(ops, name, globals()[name])
