"""TEST INFRASTRUCTURE: a plain restatement of hero_temporal_nms (include/hero_b200.h, csrc/nms.cu),
written from its contract, so the NMS flow of evalpass runs on a CPU-only box and the kernel has an
exact reference on the GPU. Each group runs the greedy loop in input (= score) order; numpy
evaluates one kept entry's IoU against the rest of its group at a time."""
import numpy as np
import torch

GROUP_CAP = 100


def _times(s, e, interval, by_clip):
    if by_clip:          # fp32, each operation rounded
        iv = np.float32(interval)
        st = s.astype(np.float32) * iv
        ed = e.astype(np.float32) * iv + iv
        return st.astype(np.float64), ed.astype(np.float64)
    return s.astype(np.float64) * interval, (e.astype(np.float64) + 1) * interval


def nms_row(score, mom, n_in, thd, interval, by_clip):
    """score (ld,) float32, mom (ld, 3) int -> indices of the kept entries in output order."""
    mom = np.asarray(mom[:n_in])
    pad = np.nonzero(mom[:, 0] < 0)[0]
    n = int(pad[0]) if len(pad) else len(mom)
    score, mom = np.asarray(score[:n]), mom[:n]
    st, ed = _times(mom[:, 1], mom[:, 2], interval, by_clip)
    if by_clip:
        _, first, inv = np.unique(mom[:, 0], return_index=True, return_inverse=True)
        grp = first[inv.reshape(-1)]
    else:
        grp = np.zeros(n, dtype=np.int64)
    kept = []
    for g in np.unique(grp):
        idx = np.nonzero(grp == g)[0]
        alive = np.ones(len(idx), dtype=bool)
        n_kept = 0
        for a in range(len(idx)):
            if not alive[a]:
                continue
            i, js = idx[a], idx[a + 1:]
            kept.append(i)
            n_kept += 1
            if n_kept == GROUP_CAP:
                break
            inter = np.maximum(0.0, np.minimum(ed[i], ed[js]) - np.maximum(st[i], st[js]))
            uni = np.maximum(ed[i], ed[js]) - np.minimum(st[i], st[js])
            iou = np.divide(inter, uni, out=np.zeros_like(inter), where=uni != 0)
            alive[a + 1:] &= ~(iou > thd)
    kept = np.array(kept, dtype=np.int64)
    if len(kept) == 0:
        return kept
    # stable sort by descending score of the groups concatenated in order of first appearance
    order = np.lexsort((kept, grp[kept], -score[kept].astype(np.float64)))
    return kept[order]


def nms_ref(score, mom, n_in, thd, interval, by_clip, n_out):
    """numpy (nq, ld) / (nq, ld, 3) -> (score (nq, n_out), mom (nq, n_out, 3)), padded 0 / -1."""
    nq = score.shape[0]
    out_s = np.zeros((nq, n_out), dtype=np.float32)
    out_m = np.full((nq, n_out, 3), -1, dtype=np.int32)
    for q in range(nq):
        k = nms_row(score[q], mom[q], n_in, thd, interval, by_clip)[:n_out]
        out_s[q, :len(k)] = score[q, k]
        out_m[q, :len(k)] = mom[q, k]
    return out_s, out_m


def temporal_nms(score, mom, n_in, thd, interval, by_clip, n_out, out_score, out_mom):
    s, m = nms_ref(score.cpu().numpy(), mom.cpu().numpy(), n_in, thd, interval, by_clip, n_out)
    out_score.copy_(torch.from_numpy(s))
    out_mom.copy_(torch.from_numpy(m))


def install(monkeypatch):
    from hero_b200 import ops
    monkeypatch.setattr(ops, "temporal_nms", temporal_nms)
