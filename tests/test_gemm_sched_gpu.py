"""The GEMM's two work-item schedules: a static stride, and dynamic items (set for the launches
of a host thread by `ops.set_gemm_shared_sms`), where CTAs claim (tile x k-split) items from a
per-stream device counter that each launch leaves at zero for the next. Every variant and tiling
must, under either schedule, give
the same bits on repeated launches (an item's arithmetic does not depend on which CTA runs it) and
match an fp32 reference; split-K accumulation must be right for every forced split count; launches
interleaved on three streams, with programmatic dependent launch, with per-launch profiling and
with HERO_SERIAL_PROFILE, must all be right; and so must a grid with fewer items than SMs.
Outputs start NaN-filled, so an item that no CTA ran fails."""
import os
import subprocess
import sys

import pytest
import torch

from .test_gemm_pingpong_gpu import _close, _dev, _rand

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(params=["static", "dynamic"])
def schedule(request):
    from hero_b200 import ops
    ops.set_gemm_shared_sms(request.param == "dynamic")
    yield request.param
    ops.set_gemm_shared_sms(False)


@pytest.fixture
def dynamic():
    from hero_b200 import ops
    ops.set_gemm_shared_sms(True)
    yield
    ops.set_gemm_shared_sms(False)


def _nan(shape, dtype=BF16):
    return torch.full(shape, float("nan"), dtype=dtype, device=_dev())


def _case(name, m, n, k):
    """(run, ref): run(block_n) launches the variant into a fresh output and returns it."""
    from hero_b200 import ops
    a, w = _rand((m, k), seed=1), _rand((n, k), 0.05, seed=2)
    # MN-major forms of the same operands; A's rows padded to a multiple of 64 in storage
    a_t = torch.zeros((k, (m + 63) // 64 * 64), dtype=BF16, device=_dev())
    a_t[:, :m] = a.t()
    a_t = a_t[:, :m]
    w_t = w.t().contiguous()
    bias = _rand((n,), 0.5, seed=3, dtype=torch.float32)
    rb = _rand((m, n), seed=4)
    rf = _rand((m, n), 2.0, seed=5, dtype=torch.float32)
    mm = a.float() @ w.float().t()
    if name == "bf16":
        return lambda bn: ops.gemm(a, w, _nan((m, n)), bias=bias, block_n=bn), mm + bias
    if name == "bf16_resid":
        return lambda bn: ops.gemm(a, w, _nan((m, n)), resid=rb, block_n=bn), mm + rb.float()
    if name == "gelu_aux":
        def run(bn):
            out, d = _nan((m, n)), _nan((m, n))
            ops.gemm(a, w, out, bias=bias, act=ops.ACT_GELU, aux_out=d, block_n=bn)
            return torch.cat([out, d], 1)
        x = mm + bias
        cdf = 0.5 * (1.0 + torch.erf(x * 0.7071067811865476))
        pdf = torch.exp(-0.5 * x * x) * 0.3989422804014327
        return run, torch.cat([x * cdf, cdf + x * pdf], 1)
    if name == "gelu":
        return (lambda bn: ops.gemm(a, w, _nan((m, n)), bias=bias, act=ops.ACT_GELU, block_n=bn),
                torch.nn.functional.gelu(mm + bias))
    if name == "relu_resid":
        return (lambda bn: ops.gemm(a, w, _nan((m, n)), resid=rb, act=ops.ACT_RELU, block_n=bn),
                torch.relu(mm) + rb.float())
    if name == "f32_store":
        return (lambda bn: ops.gemm(a, w, _nan((m, n), torch.float32), bias=bias, block_n=bn),
                mm + bias)
    if name == "f32_resid":
        return (lambda bn: ops.gemm(a, w, _nan((m, n), torch.float32), resid=rf, block_n=bn),
                mm + rf)
    if name == "f32_resid_ln":
        gamma = 1.0 + 0.1 * _rand((n,), seed=6, dtype=torch.float32)
        beta = _rand((n,), 0.2, seed=7, dtype=torch.float32)
        mean = rf.mean(-1)
        rstd = torch.rsqrt(rf.var(-1, unbiased=False) + 1e-12)
        return (lambda bn: ops.gemm(a, w, _nan((m, n), torch.float32), resid=rf,
                                    resid_ln=(mean, rstd, gamma, beta), block_n=bn),
                mm + torch.nn.functional.layer_norm(rf, (n,), gamma, beta, 1e-12))
    if name == "dgrad_bmn":
        return (lambda bn: ops.gemm(a, w_t, _nan((m, n)), b_mn=True, block_n=bn), mm)
    if name == "dgrad_bmn_resid":
        return (lambda bn: ops.gemm(a, w_t, _nan((m, n)), b_mn=True, resid=rb, block_n=bn),
                mm + rb.float())
    if name == "gelu_grad":
        return (lambda bn: ops.gemm(a, w_t, _nan((m, n)), b_mn=True, act=ops.ACT_GELU_GRAD,
                                    aux_in=rb, block_n=bn), mm * rb.float())
    if name == "ce_grad":
        labels = torch.randint(0, n, (m,), generator=torch.Generator().manual_seed(8),
                               dtype=torch.int32).to(_dev())
        lse = torch.logsumexp(mm, 1)
        g = _rand((m,), 1.0, seed=9, dtype=torch.float32)
        p = torch.softmax(mm, 1)
        p[torch.arange(m, device=_dev()), labels.long()] -= 1.0
        return (lambda bn: ops.lm_head_ce_dlogits(a, w, None, labels, lse, g, n, _nan((m, n))),
                p * g[:, None])
    if name == "ce":
        labels = torch.randint(0, n, (m,), generator=torch.Generator().manual_seed(8),
                               dtype=torch.int32).to(_dev())
        return (lambda bn: ops.ce_finish(*ops.lm_head_ce_partials(a, w, None, labels, n))[0],
                torch.logsumexp(mm, 1) - mm[torch.arange(m, device=_dev()), labels.long()])
    if name == "acc_mnmajor":     # dW += dY^T X, layout (1, 1)
        return (lambda bn: ops.gemm(a_t, w_t, torch.full((m, n), 0.5, device=_dev()), a_mn=True,
                                    b_mn=True, accumulate_f32=True, block_n=bn), 0.5 + mm)
    if name == "acc_kmajor":      # layout (0, 0)
        return (lambda bn: ops.gemm(a, w, torch.full((m, n), 0.5, device=_dev()),
                                    accumulate_f32=True, block_n=bn), 0.5 + mm)
    raise KeyError(name)


STORED = ["bf16", "bf16_resid", "gelu", "gelu_aux", "relu_resid", "f32_store", "f32_resid",
          "f32_resid_ln", "dgrad_bmn", "dgrad_bmn_resid", "gelu_grad", "ce_grad", "ce"]
ACCUMULATED = ["acc_mnmajor", "acc_kmajor"]


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("name", STORED + ACCUMULATED)
def test_every_variant_repeats_bit_for_bit_and_matches_fp32(name, bn, schedule):
    """2 000 x 768 outputs, K = 1 024: 16 row blocks, so CTAs take one or two items; a variant
    without a wide form runs its 128 x 128 form for either request."""
    run, ref = _case(name, 2000, 768, 1024)
    first = run(bn)
    _close(first, ref, 6e-2, 2e-2, f"{name} bn{bn}")
    if name in STORED:
        for _ in range(3):
            assert torch.equal(run(bn), first), f"{name} bn{bn}: not repeatable"


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("k_splits", range(1, 9))
@pytest.mark.parametrize("a_mn", [True, False])
def test_split_k_accumulation_for_forced_splits(a_mn, k_splits, bn, schedule):
    """The weight-gradient shape of the temporal encoder (K = 3 200 tokens) at every split 1..8."""
    from hero_b200 import ops
    n_out, n_in, tokens = 768, 3072, 3200
    dy, x = _rand((tokens, n_out), 0.1, seed=20), _rand((tokens, n_in), seed=21)
    ref = 0.5 + dy.float().t() @ x.float()
    out = torch.full((n_out, n_in), 0.5, device=_dev())
    if a_mn:
        ops.gemm(dy, x, out, a_mn=True, b_mn=True, accumulate_f32=True, k_splits=k_splits,
                 block_n=bn)
    else:
        ops.gemm(dy.t().contiguous(), x.t().contiguous(), out, accumulate_f32=True,
                 k_splits=k_splits, block_n=bn)
    _close(out, ref, 5e-2, 5e-3, f"split {k_splits} bn{bn} a_mn={a_mn}")


@pytest.mark.parametrize("m,n", [(100, 64), (256, 256), (1000, 512)])
@pytest.mark.parametrize("bn", [128, 256])
def test_fewer_items_than_sms(m, n, bn, schedule):
    """1, 2-4 and 8-32 items: most SMs get no CTA, and the grid is as wide as the item count."""
    for name in ("bf16", "dgrad_bmn_resid", "f32_resid_ln", "acc_mnmajor"):
        run, ref = _case(name, m, n, 256)
        _close(run(bn), ref, 6e-2, 2e-2, f"{name} {m}x{n} bn{bn}")


def interleaved_streams(rounds):
    """Three streams, each with its own sequence of stored GEMMs and split-K weight gradients that
    read the previous launch's output, so a stream whose launches overlapped or skipped an item
    would go wrong. Returns the number of mismatches against the same sequence run serially."""
    from hero_b200 import ops
    ops.set_gemm_shared_sms(True)
    m, n, k = 1536, 768, 768
    w = _rand((n, k), 0.018, seed=30)    # keeps the chained activations near unit scale
    xs = [_rand((m, k), seed=31 + i) for i in range(3)]

    def seq(x, out_acc):
        h = x
        for r in range(rounds):
            y = torch.empty((m, n), dtype=BF16, device=_dev())
            ops.gemm(h, w, y, block_n=128 if r % 2 else 256)
            y2 = torch.empty((m, n), dtype=BF16, device=_dev())
            ops.gemm(y, w.t().contiguous(), y2, b_mn=True, resid=h, block_n=256)
            ops.gemm(y2, h, out_acc, a_mn=True, b_mn=True, accumulate_f32=True,
                     k_splits=1 + r % 4, block_n=256 if r % 3 else 128)
            h = y2
        return h

    serial_acc = [torch.zeros((n, k), device=_dev()) for _ in range(3)]
    serial = [seq(xs[i], serial_acc[i]) for i in range(3)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(3)]
    accs = [torch.zeros((n, k), device=_dev()) for _ in range(3)]
    outs = [None] * 3
    torch.cuda.synchronize()
    # launches return at once, so the three streams' grids run side by side on the device
    for i in range(3):
        with torch.cuda.stream(streams[i]):
            outs[i] = seq(xs[i], accs[i])
    torch.cuda.synchronize()
    bad = 0
    for i in range(3):
        bad += int(not torch.equal(outs[i], serial[i]))
        err = (accs[i] - serial_acc[i]).abs().max().item()
        bad += int(not err <= 1e-3 * max(1.0, serial_acc[i].abs().max().item()))
    return bad


@pytest.mark.parametrize("profile", [False, True], ids=["plain", "gemm_profile"])
def test_interleaved_launches_on_three_streams(profile, dynamic):
    """3 x 40 rounds x 3 launches; programmatic dependent launch is on, and with per-launch
    profiling each launch is also bracketed by events."""
    from hero_b200 import ops
    if profile:
        ops.start_gemm_profile()
    try:
        assert interleaved_streams(40) == 0
    finally:
        if profile:
            ops.stop_gemm_profile()


def test_interleaved_launches_with_serial_profile():
    """HERO_SERIAL_PROFILE=1 (no programmatic dependent launch) is read once per process."""
    code = ("import sys; sys.path.insert(0, %r); import tests.test_gemm_sched_gpu as t; "
            "sys.exit(t.interleaved_streams(20))" % ROOT)
    env = dict(os.environ, HERO_SERIAL_PROFILE="1")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
