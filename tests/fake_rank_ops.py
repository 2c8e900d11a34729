"""TEST INFRASTRUCTURE: torch restatements of the ranking entry points of csrc/rank.cu
(include/hero_b200.h: hero_rank_topk, hero_vcmr_span_probs, hero_vcmr_moment_topn), in the style
of tests/fake_ops.py, so the retrieval orchestration runs on a CPU-only box. Ties are broken by
stable sorts (lower index first), as the kernels do. Also used on the GPU as the fp32 restatement
the kernels are checked against."""
import torch

from tests import fake_ops


def rank_topk(x, n, k, values, indices, alpha=0.0, apply_exp=False):
    v = x[:, :n].float()
    order = torch.sort(v, dim=1, descending=True, stable=True).indices[:, :k]
    top = v.gather(1, order)
    values.copy_(torch.exp(alpha * top) if apply_exp else top)
    indices.copy_(order.int())


def span_probs_ref(sim, mask_u8, w_st, w_ed):
    """(pairs, L) similarities -> start / end probabilities."""
    on = mask_u8.bool()
    st = torch.where(on, fake_ops._conv_same(sim, w_st), torch.full_like(sim, -1e4))
    ed = torch.where(on, fake_ops._conv_same(sim, w_ed), torch.full_like(sim, -1e4))
    return torch.softmax(st, -1), torch.softmax(ed, -1)


def vcmr_span_probs(s, pair_row, pair_clip, row_inv, frame_inv, mask_u8, w_st, w_ed, nv, length,
                    st, ed):
    r, c = pair_row.long(), pair_clip.long()
    cols = c[:, None] * length + torch.arange(length, device=s.device)[None, :]
    raw = s[r[:, None], cols]
    sim = raw / (row_inv.abs()[r][:, None] * frame_inv.abs()[cols])
    a, b = span_probs_ref(sim, mask_u8[c], w_st, w_ed)
    st.copy_(a)
    ed.copy_(b)


def band_mask(length, min_l, max_l, device=None):
    s = torch.arange(length, device=device)
    d = s[None, :] - s[:, None]                     # e - s
    return (d >= min_l) & (d < max_l)


def moment_topn_ref(st, ed, vf, length, min_l, max_l, n):
    """st / ed (nq, k, L), vf (nq, k) or None -> (score (nq, n), jse (nq, n, 3)), band-valid
    spans only, descending, ties to the lower flat index; padded with 0 / -1."""
    nq, k, L = st.shape
    prod = st[:, :, :, None] * (1.0 if vf is None else vf[:, :, None, None]) * ed[:, :, None, :]
    valid = band_mask(L, min_l, max_l, st.device)[None, None].expand(nq, k, L, L).reshape(nq, -1)
    flat = prod.reshape(nq, -1)
    score = torch.zeros(nq, n, dtype=torch.float32, device=st.device)
    jse = torch.full((nq, n, 3), -1, dtype=torch.int32, device=st.device)
    for q in range(nq):
        idx = torch.nonzero(valid[q]).flatten()
        vals = flat[q, idx]
        order = torch.sort(vals, descending=True, stable=True).indices[:n]
        sel = idx[order]
        c = len(sel)
        score[q, :c] = vals[order]
        jse[q, :c, 0] = (sel // (L * L)).int()
        jse[q, :c, 1] = ((sel // L) % L).int()
        jse[q, :c, 2] = (sel % L).int()
    return score, jse


def vcmr_moment_topn(st, ed, video_factor, nq, k, length, min_l, max_l, n, score, jse):
    a, b = moment_topn_ref(st.reshape(nq, k, length), ed.reshape(nq, k, length),
                           None if video_factor is None else video_factor.reshape(nq, k),
                           length, min_l, max_l, n)
    score.copy_(a)
    jse.copy_(b)


def vsm_masked_max(s, mask_u8, nq, nv, length, scores, argmax):
    """fake_ops.vsm_masked_max over the first nq rows of s only (the kernel's contract)."""
    fake_ops.vsm_masked_max(s[:nq], mask_u8, nq, nv, length, scores, argmax)


def l2norm_split(x, hi, lo, inv, eps=1e-5):
    """fake_ops.l2norm_split writing only the first x.shape[0] inverse norms (the kernel's
    contract: inv may be longer)."""
    fake_ops.l2norm_split(x, hi, lo, inv[:x.shape[0]], eps)


class QueryStager:
    """evalpass._QueryStager without a CUDA stream: host batches are ranked where they are."""

    def __init__(self, device):
        pass

    def stage(self, host_batch):
        return host_batch

    def release(self):
        pass


def install(monkeypatch):
    fake_ops.install(monkeypatch)
    from hero_b200 import evalpass, ops
    for name in ("rank_topk", "vcmr_span_probs", "vcmr_moment_topn", "vsm_masked_max",
                 "l2norm_split"):
        monkeypatch.setattr(ops, name, globals()[name])
    monkeypatch.setattr(evalpass, "_QueryStager", QueryStager)
