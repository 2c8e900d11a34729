"""Dropout-on parity of the layer runtime: the attention kernels, the LayerNorm backward's masked
copy (`drop2` / `dx_drop`) and the native BertLayer stack (`ops.bert_stack_fwd` /
`ops.bert_stack_bwd`) at p = 0.1 against float64 references that apply the same masks.

The masks are not restated from the counter hash: they are read back from the product kernels.
  element-wise sites (GEMM epilogue, LayerNorm drop2): a GEMM with A = W = 0 and bias = 1 stores
      exactly the scaled mask (keep / (1 - p), or 0);
  attention probabilities: with Q = K = 0 every row of P is uniform (1 / n over its sequence), and
      V = one-hot of the key's position (64 positions per probe) makes ctx[i, h * 64 + c] the
      dropped probability of key 64 r + c for query i in head h.
The only RNG code here is `_site_key`, the per-(layer, site) key derivation that the stack
documents in include/hero_b200.h (hero_stack_args) and implements in csrc/stack.cu.

Tolerances are those of the dropout-off tests: tests/test_kernels_gpu.py for the kernels,
SURVEY.md §8c (tests/test_bench_path_gpu.py) for the stack. Each comparison that a wrong mask
would break also has a negative control: the same reference with a wrong mask must fail it.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
P_DROP = 0.1
OUT_MAX, OUT_MEAN, OUT_COS, GRAD_REL = 6e-2, 8e-3, 0.999, 3e-2


def _dev():
    return torch.device("cuda:0")


def _rand(shape, scale=1.0, seed=0, dtype=BF16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(_dev())


def _n_bad(got, ref, atol, rtol):
    err = (got.double() - ref.double()).abs()
    return int((~(err <= atol + rtol * ref.double().abs())).sum().item())


def _close(got, ref, atol, rtol, what=""):
    """Every element within atol + rtol |ref|; NaN counts as out of tolerance."""
    bad = _n_bad(got, ref, atol, rtol)
    err = (got.double() - ref.double()).abs()
    assert bad == 0, (f"{what}: {bad}/{err.numel()} elements out of tolerance; "
                      f"max abs err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}")


# ------------------------------------------------------------------------------ mask read-back
def _elementwise_mask(m, n, drop):
    """Keep mask [m, n] of the GEMM epilogue's dropout for element (row, col) under drop =
    (threshold, key, scale): A = W = 0 and bias = 1 make the fp32 output the scaled mask."""
    from hero_b200 import ops
    a = torch.zeros(m, 64, dtype=BF16, device=_dev())
    w = torch.zeros(n, 64, dtype=BF16, device=_dev())
    bias = torch.ones(n, device=_dev())
    out = torch.full((m, n), float("nan"), device=_dev())
    ops.gemm(a, w, out, bias=bias, drop=drop)
    keep = out != 0
    # kept elements are exactly 1 * scale (an unwritten NaN fails this too)
    assert torch.equal(out[keep], torch.full_like(out[keep], drop[2])), "epilogue mask values"
    return keep


def _attention_mask(att, lens, heads, drop):
    """Keep masks of the attention kernels for the plan `att` of packed sequences `lens` under
    drop: one bool [heads, n, n] per sequence (query, key), read from the forward kernel."""
    from hero_b200 import ops
    H, ntok = heads * 64, sum(lens)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    pos = torch.from_numpy(np.concatenate([np.arange(n) for n in lens])).to(_dev())
    seq_n = torch.from_numpy(np.repeat(np.asarray(lens, np.float64), lens)).to(_dev())
    n_probe = max(1, math.ceil(max(lens) / 64))
    qkv = torch.zeros(ntok, 3 * H, dtype=BF16, device=_dev())
    ctx = torch.empty(ntok, H, dtype=BF16, device=_dev())
    probes = []
    for r in range(n_probe):
        v = torch.zeros(ntok, 64, dtype=BF16, device=_dev())
        rows = ((pos >= 64 * r) & (pos < 64 * r + 64)).nonzero().squeeze(1)
        v[rows, pos[rows] - 64 * r] = 1
        qkv[:, 2 * H:] = v.repeat(1, heads)
        ctx.fill_(float("nan"))
        ops.attn_fwd(qkv, att, ctx, heads=heads, drop=drop)
        probes.append(ctx.double().view(ntok, heads, 64))
    probe = torch.cat(probes, -1)        # [ntok, heads, 64 n_probe]: M_h[i, j] / ((1 - p) n_i)
    kept = probe != 0
    want = (drop[2] / seq_n)[:, None, None].expand_as(probe)
    # every kept entry is the scaled uniform probability, up to bf16 rounding of P and of ctx
    ratio = probe[kept] / want[kept]
    assert ratio.numel() == 0 or (ratio - 1).abs().max().item() <= 1e-2, "probe values"
    # nothing outside the query's own sequence (block-diagonal tiles) or past its length
    col = torch.arange(probe.shape[-1], device=_dev())
    assert not (kept & (col[None, None, :] >= seq_n[:, None, None])).any(), "probe leak"
    return [kept[cu[s]:cu[s + 1], :, :n].permute(1, 0, 2) for s, n in enumerate(lens)]


def _mul32(a, b):
    return (a * b) & 0xFFFFFFFF


def _site_key(base, layer, site):
    """Dropout key of (layer, site) in the layer runtime (csrc/stack.cu `site_key`); sites:
    0 = attention probabilities, 1 = attention-output dense, 2 = FFN-down dense."""
    h = base ^ _mul32(0x9E3779B1, layer * 4 + site + 1)
    h ^= h >> 16
    h = _mul32(h, 0x85EBCA6B)
    h ^= h >> 13
    h = _mul32(h, 0xC2B2AE35)
    h ^= h >> 16
    return h


def _att_plan(lens):
    from tests.test_kernels_gpu import _att_plan as plan
    return plan(lens)


def test_elementwise_mask_read_back_equals_the_epilogue_hash():
    """The read-back mask is the one tests/test_gemm_pingpong_gpu.py restates from the hash."""
    from hero_b200 import ops
    from tests.test_gemm_pingpong_gpu import _dropout_keep
    m, n = 1037, 768
    drop = ops.drop_params(P_DROP, 0xC0FFEE)
    keep = _elementwise_mask(m, n, drop)
    assert torch.equal(keep, _dropout_keep(m, n, drop[0], drop[1]))
    assert abs(keep.float().mean().item() - (1 - P_DROP)) < 0.01


# ------------------------------------------------------------------------------ attention
def _attn_ref64(qkv, lens, heads, masks=None, scale=1.0):
    """ctx = (softmax(Q K^T / 8) o M * scale) V per sequence and head, in the dtype of qkv."""
    H = heads * 64
    outs, off = [], 0
    for s, n in enumerate(lens):
        if n == 0:
            continue
        blk = qkv[off:off + n]
        q, k, v = (blk[:, i * H:(i + 1) * H].reshape(n, heads, 64).transpose(0, 1)
                   for i in range(3))
        p = torch.softmax(q @ k.transpose(1, 2) / 8.0, dim=-1)
        if masks is not None:
            p = p * masks[s].to(p.dtype) * scale
        outs.append((p @ v).transpose(0, 1).reshape(n, H))
        off += n
    return torch.cat(outs, 0)


ATT_LENS = [[25] * 40, [1, 7, 33, 64, 100, 128, 2, 90], [100] * 8, [16] * 32, [3] * 40 + [1] * 9,
            [3, 0, 5, 120, 9], [20, 200, 31, 129, 64], [514], [300, 7, 768]]


@pytest.mark.parametrize("lens", ATT_LENS)
def test_attention_dropout_fwd_bwd_vs_float64(lens):
    """ctx, dQ, dK, dV and the accumulated QKV bias gradient with dropout on, on the tile path
    (short rows, 16-sequence tiles, an empty row) and the long-row path (129 .. 768 keys)."""
    from hero_b200 import ops
    heads = 12 if max(lens) <= 200 else 3
    ntok, H = sum(lens), heads * 64
    qkv = _rand((ntok, 3 * H), 1.0, seed=500)
    sp, att = _att_plan(lens)
    assert sp.n_long == sum(n > 128 for n in lens)
    drop = ops.drop_params(P_DROP, 0x5EED0 + len(lens))
    masks = _attention_mask(att, lens, heads, drop)
    dropped = sum(int((~m).sum()) for m in masks)
    total = sum(m.numel() for m in masks)
    if total >= 20000:
        assert abs(dropped / total - P_DROP) < 0.02, dropped / total

    ctx = torch.empty(ntok, H, dtype=BF16, device=_dev())
    lse = torch.empty(ntok, heads, device=_dev())
    ops.attn_fwd(qkv, att, ctx, heads=heads, drop=drop, lse=lse)
    qr = qkv.double().requires_grad_(True)
    ref = _attn_ref64(qr, lens, heads, masks, drop[2])
    _close(ctx, ref, 2e-2, 1.6e-2, "attention fwd with dropout")
    dctx = _rand((ntok, H), 1.0, seed=501)
    ref.backward(dctx.double())
    dqkv = torch.empty_like(qkv)
    dbias = torch.full((3 * H,), 0.5, device=_dev())
    ops.attn_bwd(qkv, att, ctx, dctx, lse, dqkv, heads=heads, drop=drop, dbias=dbias)
    for i, name in enumerate(("dQ", "dK", "dV")):
        _close(dqkv[:, i * H:(i + 1) * H], qr.grad[:, i * H:(i + 1) * H], 4e-2, 3e-2,
               f"attention bwd with dropout: {name}")
    want = 0.5 + dqkv.double().sum(0)
    tol = 2e-3 * dqkv.double().abs().sum(0).max().item() + 1e-3
    assert (dbias.double() - want).abs().max().item() <= tol

    # negative control: the masks of another key break the dQ / dK comparison
    other = _attention_mask(att, lens, heads, (drop[0], drop[1] ^ 0x2545F491, drop[2]))
    qo = qkv.double().requires_grad_(True)
    _attn_ref64(qo, lens, heads, other, drop[2]).backward(dctx.double())
    for i, name in enumerate(("dQ", "dK")):
        sl = slice(i * H, (i + 1) * H)
        assert _n_bad(dqkv[:, sl], qo.grad[:, sl], 4e-2, 3e-2) > 0, \
            f"{name}: a reference with another key's mask passes too"


# ------------------------------------------------------------------------------ LayerNorm drop2
@pytest.mark.parametrize("n", [1037, 16512])
def test_ln_backward_drop2_uses_the_gemm_epilogue_mask(n):
    """The stack's LayerNorm backward: fp32 pre-LN sums, h = 768, eps 1e-12; dx_drop (the gradient
    of the dropped GEMM branch) must use the mask the GEMM epilogue applied in the forward, and
    dbias (that GEMM's bias gradient) must be the column sums of dx_drop."""
    from hero_b200 import ops
    h, eps = 768, 1e-12
    x = _rand((n, h), 2.0, seed=300, dtype=torch.float32)
    gamma = 1.0 + 0.1 * _rand((h,), 1.0, seed=301, dtype=torch.float32)
    beta = _rand((h,), 0.2, seed=302, dtype=torch.float32)
    y = torch.empty(n, h, dtype=BF16, device=_dev())
    mean, rstd = torch.empty(n, device=_dev()), torch.empty(n, device=_dev())
    ops.ln_fwd(x, gamma, beta, eps, y, n_rows=n, mean=mean, rstd=rstd)
    dy = _rand((n, h), 1.0, seed=303)
    drop2 = ops.drop_params(P_DROP, 0xD2D2 + n)
    dx = torch.full((n, h), float("nan"), dtype=BF16, device=_dev())
    dxd = torch.full((n, h), float("nan"), dtype=BF16, device=_dev())
    dgamma, dbeta, dbias = (torch.zeros(h, device=_dev()) for _ in range(3))
    ops.ln_bwd(dy, x, gamma, mean, rstd, n_rows=n, dx=dx, dx_drop=dxd, drop2=drop2,
               dgamma=dgamma, dbeta=dbeta, dbias=dbias)

    xr = x.double().requires_grad_(True)
    g, b = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    torch.nn.functional.layer_norm(xr, (h,), g, b, eps).backward(dy.double())
    _close(dx, xr.grad, 1e-2, 1.6e-2, "ln dx")

    keep = _elementwise_mask(n, h, drop2)
    assert abs(keep.float().mean().item() - (1 - P_DROP)) < 0.01
    assert int((dxd[~keep] != 0).sum()) == 0, "dx_drop is non-zero where the epilogue dropped"
    _close(dxd[keep], xr.grad[keep] * drop2[2], 1e-2 * drop2[2], 1.6e-2, "ln dx_drop (kept)")

    ref_bias = (xr.grad * keep * drop2[2]).sum(0)
    tol = 1e-4 * (xr.grad * keep * drop2[2]).abs().sum(0) + 1e-3
    assert bool(((dbias.double() - ref_bias).abs() <= tol).all()), \
        f"dbias vs column sums of dx_drop: max err {(dbias.double() - ref_bias).abs().max():.4g}"
    # ... and that is measurably not the column sums of the unmasked dx
    assert ((dbias.double() - xr.grad.sum(0)).abs() / tol).max().item() > 10
    x64 = x.double()
    xhat = (x64 - x64.mean(-1, keepdim=True)) * torch.rsqrt(x64.var(-1, unbiased=False,
                                                                    keepdim=True) + eps)
    for got, ref, terms, name in ((dgamma, g.grad, dy.double() * xhat, "dgamma"),
                                  (dbeta, b.grad, dy.double(), "dbeta")):
        err = (got.double() - ref).abs()
        assert bool((err <= 1e-4 * terms.abs().sum(0) + 1e-3).all()), \
            f"ln {name}: max err {err.max():.4g}"


# ------------------------------------------------------------------------------ BertLayer stack
N_LAYERS, HID, HEADS, INTER, EPS = 3, 768, 12, 3072, 1e-12

STACK_LAYOUTS = {
    # short rows, rows that fill the 16-sequence tile cap, and one row of each long-row size
    "ragged": [1, 7, 33, 64, 100, 128, 2, 90] + [3] * 20 + [129, 514],
    # cross-modal pass of the benchmark: 640 rows x (5 frames + 20 tokens) + 32 queries x 16
    "cross_modal_bench": [25] * 640 + [16] * 32,
    # temporal pass of the benchmark: 32 clips x 100 frames
    "temporal_bench": [100] * 32,
}

def _stack_weights(seed):
    """Seeded BertLayer weights (reference key names, fp32): matrices std 0.02, biases 0.05,
    LayerNorm gains 1 + 0.1 noise (oracle.hero_oracle.seeded_weights)."""
    from oracle import hero_oracle as orc
    shapes = orc.param_shapes(f_layers=0, c_layers=N_LAYERS)
    shapes = {k[len("c_encoder.encoder."):]: v for k, v in shapes.items()
              if k.startswith("c_encoder.encoder.layer.")}
    return orc.seeded_weights(shapes, seed=seed)


def _layer_weights(P, i):
    """functional.LayerWeights of layer i: bf16 GEMM weights, fp32 vectors, on the device."""
    from hero_b200 import functional
    p = f"layer.{i}."
    lw = functional.LayerWeights()

    def w(t):
        return t.to(BF16).contiguous().to(_dev())

    def v(t):
        return t.float().contiguous().to(_dev())

    qkv = [p + f"attention.self.{nm}." for nm in ("query", "key", "value")]
    lw.wqkv = w(torch.cat([P[k + "weight"] for k in qkv]))
    lw.bqkv = v(torch.cat([P[k + "bias"] for k in qkv]))
    lw.wo, lw.bo = w(P[p + "attention.output.dense.weight"]), v(P[p + "attention.output.dense.bias"])
    lw.ln1_g = v(P[p + "attention.output.LayerNorm.weight"])
    lw.ln1_b = v(P[p + "attention.output.LayerNorm.bias"])
    lw.w1, lw.b1 = w(P[p + "intermediate.dense.weight"]), v(P[p + "intermediate.dense.bias"])
    lw.w2, lw.b2 = w(P[p + "output.dense.weight"]), v(P[p + "output.dense.bias"])
    lw.ln2_g = v(P[p + "output.LayerNorm.weight"])
    lw.ln2_b = v(P[p + "output.LayerNorm.bias"])
    return lw


def _got_grads(grads, i):
    """The stack's gradients of layer i under the reference's parameter names."""
    g, p, H = grads[i], f"layer.{i}.", HID
    out = {}
    for j, nm in enumerate(("query", "key", "value")):
        out[p + f"attention.self.{nm}.weight"] = g["dwqkv"][j * H:(j + 1) * H]
        out[p + f"attention.self.{nm}.bias"] = g["dbqkv"][j * H:(j + 1) * H]
    for name, key in (("dwo", "attention.output.dense.weight"), ("dbo", "attention.output.dense.bias"),
                      ("dln1_g", "attention.output.LayerNorm.weight"),
                      ("dln1_b", "attention.output.LayerNorm.bias"),
                      ("dw1", "intermediate.dense.weight"), ("db1", "intermediate.dense.bias"),
                      ("dw2", "output.dense.weight"), ("db2", "output.dense.bias"),
                      ("dln2_g", "output.LayerNorm.weight"), ("dln2_b", "output.LayerNorm.bias")):
        out[p + key] = g[name]
    return out


def _grad_errors(got, ref):
    """{name: relative Frobenius error} over the parameters of `got`; the key bias (exact value
    0: softmax is invariant to a per-query constant) as |got| / |query-bias reference|."""
    errs = {}
    for k, gv in got.items():
        r = ref[k]
        if k.endswith("attention.self.key.bias"):
            errs[k] = gv.double().norm().item() / ref[k.replace("key.bias", "query.bias")].norm().item()
        else:
            errs[k] = (gv.double() - r).norm().item() / r.norm().item()
    return errs


def _reference(x_pad, valid, w_pad, P64, drops):
    """float64 BertLayer stack on the padded layout: (output, x gradient, parameter gradients) of
    loss = sum(out * w) over the valid positions."""
    from oracle import hero_oracle as orc
    Pg = {k: v.clone().requires_grad_(True) for k, v in P64.items()}
    xg = x_pad.clone().requires_grad_(True)
    add_mask = (1.0 - valid[:, None, None, :].double()) * -10000.0
    h = xg
    for i in range(N_LAYERS):
        h = orc.bert_layer(h, add_mask, Pg, f"layer.{i}.", HEADS, EPS,
                           drop=None if drops is None else drops[i])
    (h * w_pad).sum().backward()
    return h.detach(), xg.grad, {k: v.grad for k, v in Pg.items()}


def _check_out(got_pad, ref, valid, what):
    got, ref = got_pad.double()[valid], ref[valid]
    err = (got - ref).abs()
    cos = (got * ref).sum(-1) / (got.norm(dim=-1) * ref.norm(dim=-1))
    mx, mean, cmin = err.max().item(), err.mean().item(), cos.min().item()
    msg = f"{what}: max {mx:.4f} mean {mean:.5f} min-cos {cmin:.6f}"
    print(msg)
    assert mx <= OUT_MAX and mean <= OUT_MEAN and cmin >= OUT_COS, msg


def _rel(a, b):
    return (a.double() - b.double()).norm().item() / b.double().norm().item()


@pytest.mark.timeout(1500)
@pytest.mark.parametrize("p", [0.0, P_DROP], ids=["p0", "p0.1"])
@pytest.mark.parametrize("layout", list(STACK_LAYOUTS))
def test_bert_stack_fwd_bwd_vs_float64(layout, p):
    """ops.bert_stack_fwd(save=True) + ops.bert_stack_bwd over 3 layers (layers 1, 2 take the
    LayerNorm-form residual; the layer index is part of every dropout key) against the oracle's
    BertLayer in float64 with the masks the kernels applied: outputs, dx, every gradient field."""
    from hero_b200 import ops
    lens = STACK_LAYOUTS[layout]
    M, H, N, L = sum(lens), HID, len(lens), max(lens)
    valid = torch.zeros(N, L, dtype=torch.bool)
    for r, n in enumerate(lens):
        valid[r, :n] = True
    valid = valid.to(_dev())

    def to_pad(packed, fill=0.0):     # packed rows are the valid positions in row-major order
        out = torch.full((N, L) + tuple(packed.shape[1:]), fill, dtype=packed.dtype, device=_dev())
        out[valid] = packed
        return out

    P = _stack_weights(seed=21)
    layers = [_layer_weights(P, i) for i in range(N_LAYERS)]
    # the reference sees exactly what the kernels multiply: bf16-rounded GEMM weights
    P64 = {k: (v.to(BF16) if v.dim() == 2 else v).double().to(_dev()) for k, v in P.items()}
    _, att = _att_plan(lens)
    x = _rand((M, H), 1.0, seed=22)
    dout = _rand((M, H), 1.0, seed=23)
    base = 0x13579BDF
    dspec = (ops.drop_params(p, 0), ops.drop_params(p, 0), base)

    out, out_f32, saved = ops.bert_stack_fwd(x, layers, att, heads=HEADS, eps=EPS, drop=dspec,
                                             save=True)
    grads = [{k: torch.zeros(s, device=_dev()) for k, s in
              (("dwqkv", (3 * H, H)), ("dbqkv", (3 * H,)), ("dwo", (H, H)), ("dbo", (H,)),
               ("dln1_g", (H,)), ("dln1_b", (H,)), ("dw1", (INTER, H)), ("db1", (INTER,)),
               ("dw2", (H, INTER)), ("db2", (H,)), ("dln2_g", (H,)), ("dln2_b", (H,)))}
             for _ in range(N_LAYERS)]
    assert set(grads[0]) == set(ops._GRAD_FIELDS)
    dx = ops.bert_stack_bwd(x, layers, att, saved, dout, grads, heads=HEADS, eps=EPS, drop=dspec)
    torch.cuda.synchronize()

    drops = None
    if p > 0:
        hthr, _, hscale = dspec[0]
        athr, _, ascale = dspec[1]
        drops = []
        for i in range(N_LAYERS):
            am = _attention_mask(att, lens, HEADS, (athr, _site_key(base, i, 0), ascale))
            probs = torch.zeros(N, HEADS, L, L, dtype=torch.float64, device=_dev())
            for r, (n, m) in enumerate(zip(lens, am)):
                probs[r, :, :n, :n] = m.double() * ascale
            site = [to_pad(_elementwise_mask(M, H, (hthr, _site_key(base, i, s), hscale)).double()
                           * hscale) for s in (1, 2)]
            drops.append((probs, site[0], site[1]))

    x_pad, w_pad = to_pad(x.double()), to_pad(dout.double())
    ref_out, ref_dx, ref_g = _reference(x_pad, valid, w_pad, P64, drops)
    _check_out(to_pad(out_f32), ref_out, valid, f"{layout} p={p}: out_f32")
    _check_out(to_pad(out), ref_out, valid, f"{layout} p={p}: out (bf16)")
    rel_dx = _rel(dx.double(), ref_dx[valid])
    assert rel_dx <= GRAD_REL, f"{layout} p={p}: dx rel err {rel_dx:.4f}"
    bad, worst = [], (0.0, None)
    for i in range(N_LAYERS):
        for k, e in _grad_errors(_got_grads(grads, i), ref_g).items():
            lim = 2e-2 if k.endswith("key.bias") else GRAD_REL
            if e > lim:
                bad.append((k, round(e, 4)))
            if not k.endswith("key.bias") and e > worst[0]:
                worst = (e, k)
    print(f"{layout} p={p}: dx rel err {rel_dx:.4f}, worst gradient rel err {worst[0]:.4f} "
          f"({worst[1]})")
    assert not bad, f"{layout} p={p}: gradient mismatch (relative Frobenius) for {bad}"

    if layout != "ragged" or p == 0:
        return
    # Negative controls: the reference with a wrong mask misses the affected layer's gradients
    # by at least 5x the bound, so the comparison above sees this class of bug.
    wrong = {
        "layer 1 with its site-1 and site-2 masks swapped":
            (1, [drops[0], (drops[1][0], drops[1][2], drops[1][1]), drops[2]]),
        "layer 2 with the attention masks of layer 1":
            (2, [drops[0], drops[1], (drops[1][0], drops[2][1], drops[2][2])]),
        "no masks at all": (2, None),
    }
    for what, (layer, d) in wrong.items():
        _, _, g_wrong = _reference(x_pad, valid, w_pad, P64, d)
        errs = _grad_errors(_got_grads(grads, layer), g_wrong)
        e = max(v for k, v in errs.items() if not k.endswith("key.bias"))
        print(f"negative control, {what}: worst rel err of layer {layer} {e:.4f}")
        assert e >= 5 * GRAD_REL, f"{what}: layer {layer} gradients still within {e:.4f}"
