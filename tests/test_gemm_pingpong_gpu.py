"""The GEMM's fused epilogues on grids where every CTA runs several tiles: the two consumer
warpgroups alternate tiles, so an odd count per CTA leaves the second warpgroup without a last
tile, and an even count gives both the same number. Shapes follow the forward FFN-up (GELU + saved
derivative), frame_transform (ReLU + pre-activation + residual), out-projection / FFN-down
(LayerNorm-form fp32 residual + dropout) and the x GELU' dgrad with bias column sums."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
MASK32 = 0xFFFFFFFF


def _dev():
    return torch.device("cuda:0")


def _rand(shape, scale=1.0, seed=0, dtype=BF16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(_dev())


def _close(got, ref, atol, rtol, what=""):
    """Every element within atol + rtol |ref|; a NaN or unwritten (NaN-filled) element counts as bad."""
    got, ref = got.float(), ref.float()
    assert torch.isfinite(ref).all(), f"{what}: non-finite reference"
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (~(err <= tol)).sum().item()
    assert bad == 0, (f"{what}: {bad}/{err.numel()} elements out of tolerance; "
                      f"max abs err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}")


def _shape_for(tiles_per_cta):
    """(m, n) whose 128 x 128 tiles number tiles_per_cta x SMs: the persistent grid has one CTA per
    SM and each runs exactly tiles_per_cta tiles. The last row block is partial (rows past m)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = tiles_per_cta * sms
    nb = next(d for d in (6, 4, 3, 2, 1) if tiles % d == 0)
    return (tiles // nb) * 128 - 37, nb * 128


def _unwritten(m, n):
    """bf16 output filled with NaN, so that an element the kernel never writes fails _close."""
    return torch.full((m, n), float("nan"), dtype=BF16, device=_dev())


TILES_PER_CTA = [pytest.param(3, id="odd"), pytest.param(4, id="even")]


def _mul32(h, c):
    """(h * c) mod 2^32 for int64 tensors h < 2^32 and a constant c, without int64 overflow."""
    lo = h * (c & 0xFFFF)
    hi = ((h * (c >> 16)) & 0xFFFF) << 16
    return (lo + hi) & MASK32


def _hash_u32(key, idx):
    h = _mul32(idx, 0x9E3779B1) ^ key
    h ^= h >> 16
    h = _mul32(h, 0x85EBCA6B)
    h ^= h >> 13
    h = _mul32(h, 0xC2B2AE35)
    h ^= h >> 16
    return h


def _dropout_keep(m, n, threshold, key):
    """The epilogue's mask: element idx = row * n + col is kept iff its 16-bit half of
    hash(key, idx >> 1) (low half for even idx, high half for odd) is >= threshold >> 16."""
    idx = torch.arange(m * n, device=_dev(), dtype=torch.int64) & MASK32
    h = _hash_u32(key, idx >> 1)
    bits = torch.where((idx & 1) == 1, h >> 16, h & 0xFFFF)
    return (bits >= (threshold >> 16)).view(m, n)


@pytest.mark.parametrize("tiles_per_cta", TILES_PER_CTA)
def test_gemm_gelu_with_saved_derivative_many_tiles(tiles_per_cta):
    from hero_b200 import ops
    m, n = _shape_for(tiles_per_cta)
    k = 768
    a, w = _rand((m, k), seed=200), _rand((n, k), 0.05, seed=201)
    bias = _rand((n,), 0.5, seed=202, dtype=torch.float32)
    out = _unwritten(m, n)
    aux = _unwritten(m, n)
    ops.gemm(a, w, out, bias=bias, act=ops.ACT_GELU, aux_out=aux)
    pre = a.float() @ w.float().t() + bias
    dgelu = 0.5 * (1 + torch.erf(pre / math.sqrt(2))) + pre * torch.exp(-0.5 * pre * pre) / \
        math.sqrt(2 * math.pi)
    _close(out, torch.nn.functional.gelu(pre), 2e-2, 1.6e-2, f"gelu {m}x{n}")
    _close(aux, dgelu, 1e-2, 1e-2, f"saved gelu derivative {m}x{n}")


@pytest.mark.parametrize("tiles_per_cta", TILES_PER_CTA)
def test_gemm_relu_preactivation_residual_many_tiles(tiles_per_cta):
    from hero_b200 import ops
    m, n = _shape_for(tiles_per_cta)
    k = 768
    a, w = _rand((m, k), seed=210), _rand((n, k), 0.05, seed=211)
    bias = _rand((n,), 0.5, seed=212, dtype=torch.float32)
    resid = _rand((m, n), seed=213)
    out = _unwritten(m, n)
    pre = _unwritten(m, n)
    ops.gemm(a, w, out, bias=bias, act=ops.ACT_RELU, resid=resid, aux_out=pre)
    p = a.float() @ w.float().t() + bias
    _close(pre, p, 2e-2, 1.6e-2, f"saved pre-activation {m}x{n}")
    _close(out, torch.relu(p) + resid.float(), 2e-2, 1.6e-2, f"relu + residual {m}x{n}")


@pytest.mark.parametrize("tiles_per_cta", TILES_PER_CTA)
def test_gemm_layernorm_residual_with_dropout_many_tiles(tiles_per_cta):
    from hero_b200 import ops
    m, n = _shape_for(tiles_per_cta)
    k = 768
    a, w = _rand((m, k), seed=220), _rand((n, k), 0.05, seed=221)
    bias = _rand((n,), 0.5, seed=222, dtype=torch.float32)
    pre = _rand((m, n), 2.0, seed=223, dtype=torch.float32)
    gamma = 1.0 + 0.1 * _rand((n,), 1.0, seed=224, dtype=torch.float32)
    beta = _rand((n,), 0.2, seed=225, dtype=torch.float32)
    mean = pre.mean(-1)
    rstd = torch.rsqrt(pre.var(-1, unbiased=False) + 1e-12)
    drop = ops.drop_params(0.1, 777)
    out = torch.full((m, n), float("nan"), dtype=torch.float32, device=_dev())
    ops.gemm(a, w, out, bias=bias, resid=pre, resid_ln=(mean, rstd, gamma, beta), drop=drop)
    keep = _dropout_keep(m, n, drop[0], drop[1])
    assert abs(keep.float().mean().item() - 0.9) < 0.01
    v = torch.where(keep, (a.float() @ w.float().t() + bias) * drop[2], torch.zeros((), device=_dev()))
    ref = v + torch.nn.functional.layer_norm(pre, (n,), gamma, beta, 1e-12)
    _close(out, ref, 2e-3, 1e-4, f"dropout + LayerNorm-form residual {m}x{n}")


@pytest.mark.parametrize("tiles_per_cta", TILES_PER_CTA)
def test_gemm_gelu_grad_dgrad_column_sums_many_tiles(tiles_per_cta):
    from hero_b200 import ops
    m, n = _shape_for(tiles_per_cta)
    k = 768
    dy, w, dg = _rand((m, k), seed=230), _rand((k, n), 0.05, seed=231), _rand((m, n), 0.5, seed=232)
    out = _unwritten(m, n)
    cs = torch.full((n,), 0.25, device=_dev())
    ops.gemm(dy, w, out, b_mn=True, act=ops.ACT_GELU_GRAD, aux_in=dg, out_colsum=cs)
    _close(out, (dy.float() @ w.float()) * dg.float(), 2e-2, 1.6e-2, f"dgrad * saved gelu' {m}x{n}")
    want = 0.25 + out.double().sum(0)
    tol = 1e-5 * out.double().abs().sum(0).max().item() + 1e-3
    assert (cs.double() - want).abs().max().item() <= tol
