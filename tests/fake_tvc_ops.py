"""TEST INFRASTRUCTURE: torch restatement of the TVC decoder-attention entry point
(include/hero_b200.h: hero_dec_attn_fwd), in the style of tests/fake_ops.py, so HeroForTvc and
greedy decoding run on a CPU-only box. Query row i attends to the key / value rows
[kv_off[i], kv_off[i] + kv_len[i]) per head, softmax in fp32, output rounded to bf16. Also used on
the GPU as the fp32 restatement the kernel is checked against."""
import torch

from tests import fake_ops, fake_rank_ops


def dec_attn_ref(q, k, v, kv_off, kv_len, heads, head_dim=64):
    """fp32 [rows, heads * head_dim] attention output of the range contract."""
    rows = kv_off.numel() if q is None else q.shape[0]
    out = torch.empty(rows, heads * head_dim, dtype=torch.float32, device=k.device)
    off, ln = kv_off.long().tolist(), kv_len.long().tolist()
    scale = 1.0 / head_dim ** 0.5
    for i in range(rows):
        qi = q[i, :heads * head_dim].float().view(heads, 1, head_dim)
        ks = k[off[i]:off[i] + ln[i], :heads * head_dim].float().view(-1, heads, head_dim)
        vs = v[off[i]:off[i] + ln[i], :heads * head_dim].float().view(-1, heads, head_dim)
        p = torch.softmax((qi * scale) @ ks.permute(1, 2, 0), dim=-1)       # heads, 1, len
        out[i] = (p @ vs.transpose(0, 1)).reshape(-1)
    return out


def dec_attn_fwd(q, k, v, kv_off, kv_len, out, *, heads, max_kv_len, min_kv_len=1, head_dim=64):
    from hero_b200 import ops
    rows = out.shape[0]
    ops._dec_attn_bounds(rows, heads, head_dim, max_kv_len, min_kv_len)
    out[:, :heads * head_dim] = dec_attn_ref(q[:rows], k, v, kv_off[:rows], kv_len[:rows], heads,
                                             head_dim).to(out.dtype)
    return out


def install(monkeypatch):
    fake_ops.install(monkeypatch)
    from hero_b200 import ops
    monkeypatch.setattr(ops, "dec_attn_fwd", dec_attn_fwd)
    monkeypatch.setattr(ops, "rank_topk", fake_rank_ops.rank_topk)
