"""The GEMM variants with a wide (128 x 256, cooperative warpgroups) form against their 128 x 128
ping-pong form and an fp32 reference: weight gradients (split-K fp32 atomics, both layouts),
FFN-down into the fp32 residual stream (LayerNorm-form residual + dropout, plain fp32 residual),
and the dgrads with a bf16 residual (B MN-major). M = 1000 gives a partial last row block and one
tile per CTA, M = 16 512 (the step's token count) several tiles per CTA; N = 320 leaves the last
256-wide column tile partial. Outputs start NaN-filled, so an unwritten element fails. Each output
element sums K in the same k16 order in both tilings, so outputs without split-K are expected
bit-identical."""
import pytest
import torch

from .test_gemm_pingpong_gpu import _close, _dev, _dropout_keep, _rand

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
TILINGS = (128, 256)
M_ROWS = [pytest.param(1000, id="m1000"), pytest.param(16512, id="m16512")]
N_COLS = [320, 768, 2304, 3072]


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=_dev())


@pytest.mark.parametrize("tokens,n_out,k_in", [(16512, 768, 3072), (16512, 3072, 768),
                                               (16512, 2304, 768), (16512, 768, 768),
                                               (1000, 768, 320)])
@pytest.mark.parametrize("k_splits", [1, 2, 3, 7])
def test_wide_wgrad_mnmajor(tokens, n_out, k_in, k_splits):
    """dW[n_out, k_in] += dY[tokens, n_out]^T @ X[tokens, k_in] (layout (1,1), fp32 atomics)."""
    from hero_b200 import ops
    dy, x = _rand((tokens, n_out), 0.1, seed=300), _rand((tokens, k_in), seed=301)
    ref = 0.5 + dy.float().t() @ x.float()
    outs = {}
    for bn in TILINGS:
        out = torch.full((n_out, k_in), 0.5, dtype=torch.float32, device=_dev())
        ops.gemm(dy, x, out, a_mn=True, b_mn=True, accumulate_f32=True, k_splits=k_splits,
                 block_n=bn)
        _close(out, ref, 5e-2, 5e-3, f"wgrad {n_out}x{k_in} K={tokens} split {k_splits} bn{bn}")
        outs[bn] = out
    if k_splits == 1:
        assert torch.equal(outs[128], outs[256])


@pytest.mark.parametrize("n", [320, 768])
@pytest.mark.parametrize("k_splits", [1, 3])
def test_wide_wgrad_kmajor(n, k_splits):
    """Layout (0,0) fp32 accumulate (the embedding projections' weight gradients)."""
    from hero_b200 import ops
    m, k = 1000, 3200
    a, b = _rand((m, k), 0.1, seed=310), _rand((n, k), seed=311)
    ref = 0.5 + a.float() @ b.float().t()
    outs = {}
    for bn in TILINGS:
        out = torch.full((m, n), 0.5, dtype=torch.float32, device=_dev())
        ops.gemm(a, b, out, accumulate_f32=True, k_splits=k_splits, block_n=bn)
        _close(out, ref, 5e-2, 5e-3, f"wgrad k-major {m}x{n} split {k_splits} bn{bn}")
        outs[bn] = out
    if k_splits == 1:
        assert torch.equal(outs[128], outs[256])


@pytest.mark.parametrize("m", M_ROWS)
@pytest.mark.parametrize("n", N_COLS)
def test_wide_ffn_down_layernorm_residual_dropout(m, n):
    from hero_b200 import ops
    k = 3072
    a, w = _rand((m, k), seed=320), _rand((n, k), 0.02, seed=321)
    bias = _rand((n,), 0.5, seed=322, dtype=torch.float32)
    pre = _rand((m, n), 2.0, seed=323, dtype=torch.float32)
    gamma = 1.0 + 0.1 * _rand((n,), 1.0, seed=324, dtype=torch.float32)
    beta = _rand((n,), 0.2, seed=325, dtype=torch.float32)
    mean = pre.mean(-1)
    rstd = torch.rsqrt(pre.var(-1, unbiased=False) + 1e-12)
    drop = ops.drop_params(0.1, 4242)
    keep = _dropout_keep(m, n, drop[0], drop[1])
    v = torch.where(keep, (a.float() @ w.float().t() + bias) * drop[2], torch.zeros((), device=_dev()))
    ref = v + torch.nn.functional.layer_norm(pre, (n,), gamma, beta, 1e-12)
    outs = {}
    for bn in TILINGS:
        out = _nan((m, n), torch.float32)
        ops.gemm(a, w, out, bias=bias, resid=pre, resid_ln=(mean, rstd, gamma, beta), drop=drop,
                 block_n=bn)
        _close(out, ref, 2e-3, 1e-4, f"dropout + LayerNorm-form residual {m}x{n} bn{bn}")
        outs[bn] = out
    assert torch.equal(outs[128], outs[256])


@pytest.mark.parametrize("m", M_ROWS)
@pytest.mark.parametrize("n", [320, 768])
def test_wide_fp32_residual(m, n):
    from hero_b200 import ops
    k = 3072
    a, w = _rand((m, k), seed=330), _rand((n, k), 0.02, seed=331)
    bias = _rand((n,), 0.5, seed=332, dtype=torch.float32)
    resid = _rand((m, n), 2.0, seed=333, dtype=torch.float32)
    ref = a.float() @ w.float().t() + bias + resid
    outs = {}
    for bn in TILINGS:
        out = _nan((m, n), torch.float32)
        ops.gemm(a, w, out, bias=bias, resid=resid, block_n=bn)
        _close(out, ref, 2e-3, 1e-4, f"fp32 residual {m}x{n} bn{bn}")
        outs[bn] = out
    assert torch.equal(outs[128], outs[256])


@pytest.mark.parametrize("m", M_ROWS)
@pytest.mark.parametrize("n", N_COLS)
def test_wide_dgrad_bf16_residual_column_sums(m, n):
    """dX[m, n] = dY[m, k] @ W[k, n] + R (W stored [k, n]), with the column sums of dX."""
    from hero_b200 import ops
    k = 2304
    dy, w = _rand((m, k), seed=340), _rand((k, n), 0.05, seed=341)
    resid = _rand((m, n), seed=342)
    ref = dy.float() @ w.float() + resid.float()
    outs = {}
    for bn in TILINGS:
        out = _nan((m, n), BF16)
        cs = torch.full((n,), 0.25, device=_dev())
        ops.gemm(dy, w, out, b_mn=True, resid=resid, out_colsum=cs, block_n=bn)
        _close(out, ref, 2e-2, 1.6e-2, f"dgrad + bf16 residual {m}x{n} bn{bn}")
        want = 0.25 + out.double().sum(0)
        tol = 1e-5 * out.double().abs().sum(0).max().item() + 1e-3
        assert (cs.double() - want).abs().max().item() <= tol, f"column sums bn{bn}"
        outs[bn] = out
    assert torch.equal(outs[128], outs[256])
