"""TEST INFRASTRUCTURE: torch restatements of the TVC beam-search entry points
(include/hero_b200.h: hero_beam_logprob_topk, hero_beam_select, hero_dec_attn_gather_fwd), in the
style of tests/fake_tvc_ops.py, so beam search runs on a CPU-only box. Also used on the GPU as the
restatements the kernels are checked against."""
import torch

from tests import fake_tvc_ops


def dec_attn_gather_ref(q, k, v, kv_idx, kv_len, heads, head_dim=64):
    """fp32 [rows, heads * head_dim]: row i attends to the rows kv_idx[i, :kv_len[i]] of k / v."""
    rows = q.shape[0]
    out = torch.empty(rows, heads * head_dim, dtype=torch.float32, device=k.device)
    ln = kv_len[:rows].long().tolist()
    for i in range(rows):
        sel = kv_idx[i, :ln[i]].long()
        one = torch.zeros(1, dtype=torch.int32, device=k.device)
        out[i] = fake_tvc_ops.dec_attn_ref(q[i:i + 1], k[sel], v[sel], one,
                                           torch.full_like(one, ln[i]), heads, head_dim)[0]
    return out


def dec_attn_gather_fwd(q, k, v, kv_idx, kv_len, out, *, heads, max_kv_len, min_kv_len=1,
                        head_dim=64):
    rows = out.shape[0]
    out[:, :heads * head_dim] = dec_attn_gather_ref(q[:rows], k, v, kv_idx, kv_len, heads,
                                                    head_dim).to(out.dtype)
    return out


def logprob_topk_ref(x, n, beam):
    """(lse [rows], logp [rows, beam], cols [rows, beam]) in x's dtype: descending, ties to the
    lower column (a stable sort)."""
    z = x[:, :n]
    lse = torch.logsumexp(z, dim=1)
    order = torch.sort(z, dim=1, descending=True, stable=True).indices[:, :beam]
    return lse, z.gather(1, order) - lse[:, None], order


def beam_logprob_topk(x, n, beam, lse, logp, cols):
    from hero_b200 import ops
    if not 1 <= beam <= min(ops.BEAM_MAX, n) or not 1 <= n <= x.shape[1]:
        raise ValueError(f"beam_logprob_topk: beam {beam}, n {n}")
    a, b, c = logprob_topk_ref(x.float(), n, beam)
    lse.view(-1)[:x.shape[0]] = a
    logp.view(x.shape[0], beam).copy_(b)
    cols.view(x.shape[0], beam).copy_(c.int())


def select_ref(logp, cols, score, fin, length, hist, anc, *, beam, step, max_step, eos):
    """One step of the beam_select contract on host tensors: returns (score, fin, length, hist,
    anc, next_ids), each new tensor of the input's shape (hist / anc [R, max_step]; columns the
    step does not write are zero)."""
    R = score.numel()
    logp, cols = logp.reshape(R, beam).cpu(), cols.reshape(R, beam).cpu()
    score, fin, length = score.cpu(), fin.cpu(), length.cpu()
    hist, anc = hist.reshape(R, max_step).cpu(), anc.reshape(R, max_step).cpu()
    o_score, o_fin, o_len = torch.empty_like(score), torch.empty_like(fin), torch.empty_like(length)
    o_hist, o_anc = torch.zeros_like(hist), torch.zeros_like(anc)
    nxt = torch.empty(R, dtype=torch.int32)
    for n in range(R // beam):
        cand = []                                   # (score, flat index c, parent row, token)
        for p in range(beam):
            r = n * beam + p
            if fin[r]:
                cand.append((float(score[r]), p * beam, r, eos))
            else:
                for k in range(beam):
                    s = (score[r] + logp[r, k]).item()       # fp32 sum, as the kernel adds
                    cand.append((s, p * beam + k, r, int(cols[r, k])))
        cand.sort(key=lambda c: (-c[0], c[1]))
        for b, (s, _, rp, tok) in enumerate(cand[:beam]):
            r = n * beam + b
            o_score[r] = s
            o_fin[r] = int(bool(fin[rp]) or tok == eos)
            o_len[r] = length[rp] if fin[rp] else step + 1
            nxt[r] = tok
            o_hist[r, :step] = hist[rp, :step]
            o_hist[r, step] = tok
            o_anc[r, :step + 1] = anc[rp, :step + 1]
            if step + 1 < max_step:
                o_anc[r, step + 1] = (step + 1) * R + r
    return o_score, o_fin, o_len, o_hist, o_anc, nxt


def beam_select(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, *, beam, step,
                max_step, eos):
    from hero_b200 import ops
    R = logp.shape[0]
    if not 1 <= beam <= ops.BEAM_MAX or R % beam or not 0 <= step < max_step:
        raise ValueError(f"beam_select: beam {beam}, step {step} of {max_step}")
    s, f, ln, h, a, nxt = select_ref(logp, cols, *state_in, anc_in, beam=beam, step=step,
                                     max_step=max_step, eos=eos)
    o_score, o_fin, o_len, o_hist = state_out
    o_score.copy_(s)
    o_fin.copy_(f)
    o_len.copy_(ln)
    o_hist.view(R, max_step)[:, :step + 1] = h[:, :step + 1].to(o_hist.device)
    anc_out.view(R, max_step)[:, :min(step + 2, max_step)] = a[:, :min(step + 2, max_step)].to(
        anc_out.device)
    next_ids.copy_(nxt)


def install(monkeypatch):
    fake_tvc_ops.install(monkeypatch)
    from hero_b200 import ops
    for name in ("dec_attn_gather_fwd", "beam_logprob_topk", "beam_select"):
        monkeypatch.setattr(ops, name, globals()[name])
