"""CPU companions of test_attention_gpu.py: its float64 reference is the plain masked attention of
torch, its bounds are tighter on the long path than on the tile path, and the plan-edge cases of
its dispatch matrix produce the tiles they are named after."""
import math

import numpy as np
import torch

from hero_b200.plan import SeqPlan
from tests.test_attention_gpu import SCALE, _host, _reference

F64 = torch.float64


def _qkv(n_tok, heads, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(n_tok, 3 * heads * 64, generator=g, dtype=F64).to(torch.bfloat16)
    dctx = torch.randn(n_tok, heads * 64, generator=g, dtype=F64).to(torch.bfloat16)
    return qkv, dctx


def _plan(lens):
    mask = np.zeros((len(lens), max(lens)), np.int64)
    for r, n in enumerate(lens):
        mask[r, :n] = 1
    return SeqPlan(mask)


def test_reference_equals_sdpa_with_a_block_mask():
    """ctx, lse and every gradient of the per-tile reference equal float64
    scaled_dot_product_attention over the whole packed stream with a boolean block-diagonal mask."""
    heads, lens = 2, [3, 0, 17, 128, 1, 140, 60]
    sp = _plan(lens)
    hp = _host(sp)
    n, H = sp.n_tok, heads * 64
    qkv, dctx = _qkv(n, heads, 1)
    ctx0 = _reference(qkv, hp, heads)["ctx"]
    ref = _reference(qkv, hp, heads, dctx, ctx0.to(torch.bfloat16))
    X = qkv.double().requires_grad_(True)
    q, k, v = (X[:, i * H:(i + 1) * H].reshape(n, heads, 64).transpose(0, 1) for i in range(3))
    seq = torch.as_tensor(sp.seq_lo)
    mask = seq[:, None] == seq[None, :]
    out = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=SCALE)
    out.backward(dctx.double().reshape(n, heads, 64).transpose(0, 1))
    ctx = out.detach().transpose(0, 1).reshape(n, H)
    s = (q @ k.transpose(-1, -2) * SCALE).masked_fill(~mask, -math.inf)
    lse = (torch.logsumexp(s, -1) / math.log(2)).detach().t()
    assert torch.allclose(ref["ctx"], ctx, rtol=0, atol=1e-12)
    assert torch.allclose(ref["lse"], lse, rtol=0, atol=1e-12)
    assert torch.allclose(ref["dqkv"], X.grad, rtol=0, atol=1e-12)


def test_long_bounds_are_tighter_than_tile_bounds():
    """On a long sequence the long path's bounds (fp32 P and dS) sit far inside the bounds the tile
    path (bf16 P and dS) would get on the same rows: a long kernel that rounded like the tile
    kernel would be caught."""
    heads = 2
    sp = _plan([200, 5])
    hp = _host(sp)
    qkv, dctx = _qkv(sp.n_tok, heads, 2)
    ctx = _reference(qkv, hp, heads)["ctx"].to(torch.bfloat16)
    lo = _reference(qkv, hp, heads, dctx, ctx)
    hi = _reference(qkv, hp, heads, dctx, ctx, tile_bounds=True)
    rows = slice(0, 200)                 # the 200-token sequence: its own (long) tile
    for k in ("e_ctx", "tol_lse", "e_dqkv"):
        a, b = lo[k][rows], hi[k][rows]
        assert bool((a <= b).all()), k
        assert a.sum().item() < 0.2 * b.sum().item(), (k, a.sum().item(), b.sum().item())


def test_plan_edges_produce_the_intended_tiles():
    def tiles(lens):
        sp = _plan(lens)
        return sp.tile_ntok.tolist(), sp.n_long, sp.max_long

    assert tiles([8] * 16) == ([128], 0, 0)                  # 128 tokens in 16 sequences
    assert tiles([7] * 17) == ([112, 7], 0, 0)               # the 17th opens a new tile
    assert tiles([127, 1]) == ([128], 0, 0)
    assert tiles([1]) == ([1], 0, 0)
    assert tiles([63, 65, 64, 64, 0, 3]) == ([128, 128, 3], 0, 0)
    for n in (129, 256, 257, 767, 768):
        assert tiles([n]) == ([n], 1, n)
    assert tiles([20, 200, 31, 129, 64, 768, 1, 127]) == ([20, 31, 64, 128, 200, 129, 768], 3, 768)
    assert tiles([100] * 40 + [5] * 7) == ([100] * 39 + [125, 10], 0, 0)
    assert tiles([300] * 12 + [9]) == ([9] + [300] * 12, 12, 300)


def test_joint_plan_puts_long_tiles_after_both_short_streams():
    from tests.test_attention_gpu import _host_joint, _joint_with_long
    jp = _joint_with_long()
    hp = _host_joint(jp)
    ntok = np.asarray(hp["ntok"])
    tok0 = np.asarray(hp["tok0"])
    n_short = len(ntok) - hp["n_long"]
    assert hp["n_long"] == 2 and jp.max_long == 140
    assert (ntok[:n_short] <= 128).all() and (ntok[n_short:] > 128).all()
    # the query stream's short tiles (tokens >= n_video_tok) come before the video's long tiles
    assert (tok0[:n_short] >= jp.n_video_tok).any()
    assert (tok0[n_short:] < jp.n_video_tok).all()
    assert int(ntok.sum()) == jp.n_tok
