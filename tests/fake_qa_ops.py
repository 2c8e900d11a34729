"""TEST INFRASTRUCTURE: torch restatements of the video QA pooling entry points of csrc/qa.cu
(include/hero_b200.h: hero_qa_pool_fwd, hero_qa_pool_bwd), in the style of tests/fake_ops.py, so
HeroForVideoQA runs on a CPU-only box. The expressions are those of model/videoQA.py:36-59 on the
(Nv, Nq, L, H) tensor gathered through the frame map (zeros where it is -1). Also used on the GPU
as the fp32 restatement the kernels are checked against."""
import torch

from tests import fake_ops


def padded(h, frame_map, nv, nq, length):
    m = frame_map.long()
    x = torch.where((m >= 0)[:, None], h[m.clamp(min=0)], torch.zeros((), dtype=h.dtype))
    return x.view(nv, nq, length, h.shape[1])


def pool_ref(x, mask, w_qa, w_st):
    """model/videoQA.py:36-59 on x (Nv, Nq, L, H), mask (Nv, Nq, L): (st_pooled, qa_pooled, a, b)."""
    m = mask.unsqueeze(-1)
    st = torch.softmax((x @ w_st.reshape(-1, 1)) * m + (1 - m) * -1e4, dim=1)
    qa = torch.softmax((x @ w_qa.reshape(-1, 1)) * m + (1 - m) * -1e4, dim=2)
    st_pooled = torch.einsum("vqlm,vqld->vlmd", st, x).squeeze(2)
    qa_pooled = torch.einsum("vqlm,vqld->vqmd", qa, x).squeeze(2)
    return st_pooled, qa_pooled, qa.reshape(-1), st.reshape(-1)


def qa_pool_fwd(h, frame_map, mask, w_qa, w_st, nv, nq, length, a, b, qa_pooled, st_pooled):
    from hero_b200 import ops
    ops._qa_bounds(nv, nq, length, h.shape[1])
    x = padded(h, frame_map, nv, nq, length)
    sp, qp, pa, pb = pool_ref(x, mask.view(nv, nq, length), w_qa, w_st)
    a.copy_(pa)
    b.copy_(pb)
    qa_pooled.copy_(qp.reshape(nv * nq, -1))
    st_pooled.copy_(sp.reshape(nv * length, -1))


def qa_pool_bwd(h, frame_map, mask, w_qa, w_st, a, b, d_qa, d_st, nv, nq, length, dh, dw_qa,
                dw_st):
    from hero_b200 import ops
    ops._qa_bounds(nv, nq, length, h.shape[1])
    with torch.enable_grad():
        x = padded(h, frame_map, nv, nq, length).detach().requires_grad_(True)
        wq = w_qa.detach().clone().requires_grad_(True)
        ws = w_st.detach().clone().requires_grad_(True)
        sp, qp, _, _ = pool_ref(x, mask.view(nv, nq, length), wq, ws)
        torch.autograd.backward([qp.reshape(nv * nq, -1), sp.reshape(nv * length, -1)],
                                [d_qa, d_st])
    m = frame_map.long()
    keep = m >= 0
    dh[m[keep]] = x.grad.reshape(-1, h.shape[1])[keep]
    dw_qa.add_(wq.grad)
    dw_st.add_(ws.grad)


def install(monkeypatch):
    fake_ops.install(monkeypatch)
    from hero_b200 import ops
    for name in ("qa_pool_fwd", "qa_pool_bwd"):
        monkeypatch.setattr(ops, name, globals()[name])
