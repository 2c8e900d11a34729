"""The attention kernels of csrc/attention_tc.cu against float64: every path that `hero_attn_fwd` /
`hero_attn_bwd` choose between, the edges of the tile plan, exact probes, score magnitudes, the
log-sum-exp contract, the bytes the kernels may read and write, and the plans the model builds.

Paths (the short tiles of a plan come first and run on the tensor cores; the `n_long` tiles of
one sequence longer than 128 tokens come last and run on the CUDA cores):
  A1 attn_tc_fwd_kernel                          forward of a tile of <= 128 tokens, <= 16 sequences
  A2 attn_long_q_kernel<0>                       forward of one sequence of 129 ... 768 tokens
  B1 attn_tc_bwd_kernel                          backward of a tile
  B2 attn_long_q_kernel<1> + attn_long_kv_kernel backward of a long sequence (dQ; dK, dV)

Reference. include/hero_b200.h restated in float64 on the exact bf16 tensors the kernels read: per
sequence S = Q K^T / 8, P = softmax(S) over the row's own sequence, ctx = P V, lse =
logsumexp(S) / ln 2 (the log2-domain log-sum-exp of the scaled scores), and the backward by
autograd through that expression. It is built per tile with a block-diagonal mask and batched on
the device; long sequences are tiles of their own.

Every case runs on NaN-filled outputs with NaN guard rows after n_tok, behind qkv and dctx as well:
every valid element must be finite and every guard row must stay NaN (nothing may write or read
past n_tok, and an output row the kernel forgets to write stays NaN).

Tolerances, per element and per path. u = 2^-24; g(k) = k 2^-23 is the error of a k-term fp32
sum, rounding or truncating (tensor-core accumulation included); s = 1/8 the score scale, c = s /
ln 2 (scale_log2); t = 1 on the tile paths and 0 on the long paths; L = 128 on the tile paths and
n on the long ones (terms of the P V, dS K, dS^T Q and P^T dO sums); A_ij = sum_d |q_id k_jd|.
A bf16 output within e of its float64 value ref is checked as |got - ref| <= e + h(|ref| + e),
h(x) the half-ulp of bf16 at x (2^-9 to 2^-8 relative: round to nearest).
  score     raw error of S_ij: t 2^-9 + g(64) A_ij. The tile kernels add the membership shift 16384
            to the row's own scores inside the MMA; next to 16384 an fp32 score carries up to 2^-9
            absolute error while |S| < 2^13 (the raw scores of these tests stay below 2^10, and
            below 8000 where a neighbouring sequence's are larger); the long kernels use plain
            fp32 dot products.
  e_ij      = s (t 2^-9 + g(64) A_ij) + 2^-21: relative error of one forward probability (the
            row's common factors, its max and the rounding of -max c, cancel in ctx).
  ctx       e = sum_j p_j e_ij (|v_j| + |ctx|) + (t 2^-8 + g(L)) sum_j p_j |v_j| + g(L + 2) |ctx|:
            the tile forward rounds P to bf16 for P V (2^-8 relative) but takes the sum and its
            inverse from the unrounded fp32 values; the long forward keeps p in fp32.
  lse       c (t 2^-9 + g(64) max_j A_ij) + (max_j e_ij + g(L)) / ln 2 + t 2^-13 + 2^-22 (2 + |lse|)
            in log2 units: the error of the row max, of log2(sum), and on the tile path the
            rounding of -max c next to 16384 c ~ 2955 (half-ulp 2^-13).
  p (bwd)   r_ij = s (t 2^-9 + g(64) A_ij) + ln 2 (lse_i + t 2^-13) + 2^-21: relative error of the
            probability rebuilt from the stored lse (the tile path adds back 16384 c, rounded to
            2^-13 while lse < 1140).
  D_i       dO_i . O_i from the STORED bf16 ctx on both paths: dD_i = |dO_i . (ctx_stored -
            ctx_ref)_i| + g(64) sum_d |dO_id O_id|.
  dS        E_ij = p_ij ((r_ij + t 2^-8 + 2^-21) |dP_ij - D_i| + g(64) sum_d |dO_id v_jd| + dD_i):
            the tile backward rounds dS to bf16 (2^-8), the long backward keeps it in fp32.
  dQ, dK    e = s (E |K| + g(L) |dS| |K|) and s (E^T |Q| + g(L) |dS|^T |Q|).
  dV        e = F^T |dO| + g(L) P^T |dO|, F_ij = p_ij (r_ij + t 2^-8): the tile backward rounds P
            to bf16 for dV, the long backward does not. The long bounds are therefore tighter than
            the tile bounds by the 2^-8 terms (checked in test_attention_cpu.py), and a long path
            that rounded like the tile path fails them (test_negative_controls).
  dbias     per column: the float64 sum of the STORED bf16 dqkv rows plus the initial value,
            within g(128 + N) (|init| + sum_rows |dqkv|): tile sums of <= 128 terms in the MMA and
            one fp32 atomic per tile, one atomic per row on the long path (N = short tiles + long
            tokens). One wrong column cannot hide behind the largest.

Negative controls (test_negative_controls) run each check against a perturbed reference, which
must fail: one key removed from one sequence (ctx, dqkv), lse shifted by 2^-6, two dbias columns
swapped, and on a long sequence the tile path's rounding of P.

Score envelope of the magnitude tests: scaled scores spread over +-60, a common raw offset of 960,
and neighbouring sequences of a tile whose scores are 8000 raw above the row's own, half the
16384 margin of the membership shift. Nothing here goes further.
"""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from tests.test_kernels_gpu import _att_plan
from tests.test_rowwise_gpu import _n_bad, _within

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
NAN = float("nan")
LN2 = math.log(2.0)
SCALE = 0.125
SCALE_LOG2 = SCALE / LN2
GUARD = 3

FWD_KERNELS = {"A1": "attn_tc_fwd_kernel", "A2": "attn_long_q_kernel<0>"}
BWD_KERNELS = {"B1": ("attn_tc_bwd_kernel",), "B2": ("attn_long_q_kernel<1>", "attn_long_kv_kernel")}


def _dev():
    return torch.device("cuda:0")


def g(k):
    """Error of a k-term fp32 sum, relative to the sum of the magnitudes."""
    return k * 2.0 ** -23


def _half_ulp(x):
    """Half an ulp of bf16 at x >= 0 (0 at 0)."""
    _, e = torch.frexp(x)
    return torch.where(x > 0, torch.ldexp(torch.ones_like(x), e - 9), torch.zeros_like(x))


def _tol_bf16(ref, e):
    return e + _half_ulp(ref.abs() + e)


# ------------------------------------------------------------------------------ plans
def _host(sp):
    """Host copy of a SeqPlan's attention plan."""
    return {"tok0": sp.tile_tok0, "ntok": sp.tile_ntok, "n_long": int(sp.n_long),
            "seq_lo": sp.seq_lo, "n_tok": int(sp.n_tok)}


def _host_joint(jp):
    a = jp.arr
    return {"tok0": a["j_tile_tok0"], "ntok": a["j_tile_ntok"], "n_long": int(jp.n_long),
            "seq_lo": a["j_seq_lo"], "n_tok": int(jp.n_tok)}


def _lens_plan(lens):
    sp, att = _att_plan(lens)
    return _host(sp), att


def _seq_plan(sp):
    from hero_b200.plan import DeviceIndex
    dev = DeviceIndex(sp.arrays("s_"), _dev())
    return _host(sp), sp.attn(dev, "s_")


def _paths(hp):
    n_long = hp["n_long"]
    n_short = len(hp["tok0"]) - n_long
    return (({"A1"} if n_short else set()) | ({"A2"} if n_long else set()),
            ({"B1"} if n_short else set()) | ({"B2"} if n_long else set()))


# ------------------------------------------------------------------------------ float64 reference
def _groups(hp, chunk=48):
    """Token-index batches [T, L] (-1 past a tile's end): the short tiles padded to 128, in chunks,
    then each long tile alone. Yields (index, long?)."""
    tok0, ntok = np.asarray(hp["tok0"], np.int64), np.asarray(hp["ntok"], np.int64)
    n_short = len(tok0) - hp["n_long"]
    ar = np.arange(128)
    for a in range(0, n_short, chunk):
        b = min(a + chunk, n_short)
        t0, tn = tok0[a:b], ntok[a:b]
        yield np.where(ar[None] < tn[:, None], t0[:, None] + ar[None], -1), False
    for t in range(n_short, len(tok0)):
        yield (tok0[t] + np.arange(ntok[t]))[None], True


def _reference(qkv, hp, heads, dctx=None, ctx_got=None, *, drop_key=None, tile_bounds=False,
               round_p=False):
    """float64 forward (ctx, lse) and autograd backward (dqkv) of the plan hp on qkv[:n_tok], with
    the error bounds of the docstring: e_ctx, tol_lse, e_dqkv (pre-rounding parts of the bf16
    outputs). The backward needs dctx and the kernel's stored ctx. drop_key: a token whose key is
    removed from its sequence (negative control); tile_bounds: bound every tile, long ones too, as
    the tile path does; round_p: P rounded to bf16 for P V and P^T dO (the tile path's rounding)."""
    dev = qkv.device
    n_tok, H = hp["n_tok"], heads * 64
    X = qkv[:n_tok].double().requires_grad_(dctx is not None)
    seq = torch.as_tensor(np.asarray(hp["seq_lo"], np.int64), device=dev)
    r = {k: torch.zeros(n_tok, w, dtype=F64, device=dev) for k, w in
         (("ctx", H), ("e_ctx", H), ("lse", heads), ("tol_lse", heads), ("e_dqkv", 3 * H))}
    for idx_np, is_long in _groups(hp):
        idx = torch.as_tensor(idx_np, device=dev)
        T, L = idx.shape
        valid = idx >= 0
        ix = idx.clamp(min=0)
        t = 0.0 if is_long and not tile_bounds else 1.0
        nl = L if is_long else 128
        sq = torch.where(valid, seq[ix], -1)
        same = (sq[:, :, None] == sq[:, None, :]) & valid[:, :, None] & valid[:, None, :]
        if drop_key is not None:
            same &= (idx != drop_key)[:, None, :]
        eye = torch.eye(L, dtype=torch.bool, device=dev)[None]
        allow = (same | (~valid[:, :, None] & eye))[:, None]      # padding rows see themselves
        rows = X[ix]
        Q, K, V = (rows[..., i * H:(i + 1) * H].reshape(T, L, heads, 64).transpose(1, 2)
                   for i in range(3))
        S = (Q @ K.transpose(-1, -2) * SCALE).masked_fill(~allow, -math.inf)
        P = torch.softmax(S, -1)
        Pm = P.to(BF16).double() if round_p else P
        O = Pm @ V
        lse = torch.logsumexp(S, -1) / LN2
        with torch.no_grad():
            Pd, Od = P.detach(), O.detach()
            Qa, Ka, Va = Q.detach().abs(), K.detach().abs(), V.detach().abs()
            A = (Qa @ Ka.transpose(-1, -2)) * allow
            maxA = A.amax(-1)
            eps = (SCALE * (t * 2.0 ** -9 + g(64) * A) + 2.0 ** -21) * allow
            PE = Pd * eps
            PV = Pd @ Va
            e_ctx = PE @ Va + Od.abs() * PE.sum(-1, keepdim=True) + (t * 2.0 ** -8 + g(nl)) * PV \
                + g(nl + 2) * Od.abs()
            tol_lse = SCALE_LOG2 * (t * 2.0 ** -9 + g(64) * maxA) + \
                (eps.amax(-1) + g(nl)) / LN2 + t * 2.0 ** -13 + 2.0 ** -22 * (2 + lse.detach().abs())

        def put(name, val, cols=None):
            v = val.transpose(1, 2).reshape(T, L, -1)[valid]
            if cols is None:
                r[name][idx[valid]] = v
            else:
                r[name][idx[valid], cols] = v

        put("ctx", Od)
        put("e_ctx", e_ctx)
        put("lse", lse.detach().unsqueeze(-1))
        put("tol_lse", tol_lse.unsqueeze(-1))
        if dctx is None:
            continue
        dO = (dctx[ix].double() * valid[..., None]).reshape(T, L, heads, 64).transpose(1, 2)
        (O * dO).sum().backward()
        with torch.no_grad():
            Og = ctx_got[ix].double().reshape(T, L, heads, 64).transpose(1, 2)
            dOa = dO.abs()
            dP = dO @ V.detach().transpose(-1, -2)
            D = (dO * Od).sum(-1, keepdim=True)
            dD = (dO * (Og - Od)).sum(-1, keepdim=True).abs() + g(64) * (dOa * Og.abs()).sum(-1, keepdim=True)
            rp = (SCALE * (t * 2.0 ** -9 + g(64) * A) + LN2 * (tol_lse[..., None] + t * 2.0 ** -13)
                  + 2.0 ** -21)
            dS = (Pd * (dP - D)).abs()
            E = Pd * ((rp + t * 2.0 ** -8 + 2.0 ** -21) * (dP - D).abs()
                      + g(64) * (dOa @ Va.transpose(-1, -2)) + dD)
            F = Pd * (rp + t * 2.0 ** -8)
            e_dq = SCALE * ((E + g(nl) * dS) @ Ka)
            e_dk = SCALE * ((E + g(nl) * dS).transpose(-1, -2) @ Qa)
            e_dv = (F + g(nl) * Pd).transpose(-1, -2) @ dOa
            for i, e in enumerate((e_dq, e_dk, e_dv)):
                v = e.transpose(1, 2).reshape(T, L, H)[valid]
                r["e_dqkv"][idx[valid], i * H:(i + 1) * H] = v
    r["dqkv"] = X.grad if dctx is not None else None
    return r


# ------------------------------------------------------------------------------ launching
def _nan(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=_dev())


def _guarded(x):
    """x copied into the first rows of a buffer whose GUARD last rows are NaN; returns (view, buf)."""
    buf = _nan((x.shape[0] + GUARD,) + tuple(x.shape[1:]), x.dtype)
    buf[:x.shape[0]] = x
    return buf[:x.shape[0]], buf


def _inputs(hp, heads, seed):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    n, H = hp["n_tok"], heads * 64
    qkv = torch.randn(n, 3 * H, generator=gen, dtype=F64).to(BF16).to(_dev())
    dctx = torch.randn(n, H, generator=gen, dtype=F64).to(BF16).to(_dev())
    return qkv, dctx


def _launch(qkv, att, heads, dctx, *, lse_in=None, dbias0=0.5):
    """Forward and backward into NaN buffers with guard rows; qkv and dctx are read from buffers
    whose guard rows are NaN. Returns the outputs (row views) and the buffers."""
    from hero_b200 import ops
    n, H = att["n_tok"], heads * 64
    qkv_v, qkv_b = _guarded(qkv)
    dctx_v, dctx_b = _guarded(dctx)
    ctx_b, dqkv_b = _nan((n + GUARD, H), BF16), _nan((n + GUARD, 3 * H), BF16)
    lse_b = _nan(((n + GUARD) * heads,), F32)
    ctx, dqkv, lse = ctx_b[:n], dqkv_b[:n], lse_b[:n * heads].view(n, heads)
    ops.attn_fwd(qkv_v, att, ctx, heads=heads, lse=lse)
    dbias = torch.full((3 * H,), dbias0, dtype=F32, device=_dev())
    lse_b_in = lse if lse_in is None else lse_in
    ops.attn_bwd(qkv_v, att, ctx, dctx_v, lse_b_in, dqkv, heads=heads, dbias=dbias)
    torch.cuda.synchronize()
    return {"ctx": ctx, "lse": lse, "dqkv": dqkv, "dbias": dbias, "dbias0": dbias0,
            "bufs": (qkv_b, dctx_b, ctx_b, lse_b, dqkv_b)}


def _check_bytes(out, n, heads, what):
    qkv_b, dctx_b, ctx_b, lse_b, dqkv_b = out["bufs"]
    for name, b, valid in (("ctx", ctx_b, ctx_b[:n]), ("lse", lse_b, lse_b[:n * heads]),
                           ("dqkv", dqkv_b, dqkv_b[:n])):
        assert bool(torch.isfinite(valid.float()).all()), f"{what}: {name} has non-finite values"
        assert bool(torch.isnan(b[valid.shape[0]:].float()).all()), f"{what}: {name} guard written"
    for name, b in (("qkv", qkv_b), ("dctx", dctx_b)):
        assert bool(torch.isnan(b[n:].float()).all()), f"{what}: {name} guard changed"


def _dbias_tol(hp, dqkv, dbias0):
    n_short = len(hp["tok0"]) - hp["n_long"]
    n_adds = n_short + int(np.asarray(hp["ntok"])[n_short:].sum())
    return g(128 + n_adds) * (abs(dbias0) + dqkv.double().abs().sum(0))


def _check(out, ref, hp, heads, what, *, lse=True):
    H = heads * 64
    _within(out["ctx"], ref["ctx"], _tol_bf16(ref["ctx"], ref["e_ctx"]), f"{what}: ctx")
    if lse:
        _within(out["lse"], ref["lse"], ref["tol_lse"], f"{what}: lse")
    for i, name in enumerate(("dQ", "dK", "dV")):
        cols = slice(i * H, (i + 1) * H)
        _within(out["dqkv"][:, cols], ref["dqkv"][:, cols],
                _tol_bf16(ref["dqkv"][:, cols], ref["e_dqkv"][:, cols]), f"{what}: {name}")
    want = out["dbias0"] + out["dqkv"].double().sum(0)
    _within(out["dbias"], want, _dbias_tol(hp, out["dqkv"], out["dbias0"]), f"{what}: dbias")


def _run(hp, att, heads, qkv, dctx, what, **kw):
    out = _launch(qkv, att, heads, dctx, **kw)
    _check_bytes(out, hp["n_tok"], heads, what)
    ref = _reference(qkv, hp, heads, dctx, out["ctx"])
    _check(out, ref, hp, heads, what)
    return out, ref


# ------------------------------------------------------------------------------ 1. dispatch matrix
MATRIX = [  # (name, sequence lengths, heads)
    ("tile128-16seq", [8] * 16, (1, 2, 12)),
    ("16seq-then-17th", [7] * 17, (1, 12)),
    ("127+1", [127, 1], (1, 2, 12)),
    ("one-token", [1], (1, 12)),
    ("63", [63], (2,)), ("64", [64], (2,)), ("65", [65], (2,)),
    ("63-65-64-64", [63, 65, 64, 64, 0, 3], (1, 12)),
    ("long129", [129], (1, 12)), ("long256", [256], (2,)), ("long257", [257], (1, 12)),
    ("long767", [767], (1, 12)), ("long768", [768], (1, 2, 12)),
    ("mixed", [20, 200, 31, 129, 64, 768, 1, 127], (1, 2, 12)),
    ("many-tiles", [100] * 40 + [5] * 7, (12,)),           # 41 tiles x 12 heads: several waves
    ("many-long", [300] * 12 + [9], (12,)),                 # 12 long rows x 12 heads > 132 SMs
]
MATRIX_CASES = [(n, lens, h) for n, lens, hs in MATRIX for h in hs]


@pytest.mark.parametrize("name,lens,heads", MATRIX_CASES,
                         ids=[f"{n}-h{h}" for n, _, h in MATRIX_CASES])
def test_dispatch_matrix(name, lens, heads):
    hp, att = _lens_plan(lens)
    qkv, dctx = _inputs(hp, heads, seed=sum(lens) + heads)
    _run(hp, att, heads, qkv, dctx, f"{name} heads={heads}")


def _joint_with_long():
    """A JointPlan whose video stream has sequences of 140 and 129 tokens (long tiles, placed after
    the query stream's short tiles) beside short ones."""
    from hero_b200 import synth
    from hero_b200.plan import build_plans, plan_inputs
    gen = torch.Generator().manual_seed(11)
    clips = [synth.make_clip(gen, 120, [range(0, 100), range(100, 120)], [40, 10], vfeat_dim=8),
             synth.make_clip(gen, 30, [range(0, 9), range(9, 30)], [120, 6], vfeat_dim=8)]
    vb = synth.video_batch(clips)
    qb = synth.query_batch(gen, [16, 5, 30])
    rplan, _ = build_plans(plan_inputs(vb), plan_inputs(qb, "txt"))
    return rplan._joint


def _joint_case(jp):
    from hero_b200.plan import DeviceIndex
    dev = DeviceIndex(jp.arr, _dev())
    return _host_joint(jp), jp.attn(dev)


@pytest.mark.parametrize("heads", [2, 12])
def test_joint_plan_long_tiles_after_both_short_streams(heads):
    jp = _joint_with_long()
    hp, att = _joint_case(jp)
    assert hp["n_long"] == 2
    qkv, dctx = _inputs(hp, heads, seed=5 + heads)
    _run(hp, att, heads, qkv, dctx, f"joint plan heads={heads}")


def _kernel_sequence():
    """The attention kernels every profiler case launches, in launch order: all cases run in ONE
    profiler session with idle margins at both ends. Kineto maps GPU timestamps onto the host
    clock with an offset that grows with the time since the process's first profiler session
    (measured on an H100: 0.1 to 100 ms after a few minutes), and drops kernels that fall outside
    the session's window: short sessions late in a long process lose their kernels."""
    from torch.profiler import ProfilerActivity, profile

    from hero_b200 import ops
    runs = []
    for lens in [lens for _, lens, _ in MATRIX] + [None]:
        hp, att = _lens_plan(lens) if lens is not None else _joint_case(_joint_with_long())
        qkv, dctx = _inputs(hp, 2, seed=1)
        n = hp["n_tok"]
        runs.append((qkv, att, dctx, torch.empty(n, 128, dtype=BF16, device=_dev()),
                     torch.empty(n, 2, device=_dev()), torch.empty_like(qkv)))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.5)
        for qkv, att, dctx, ctx, lse, dqkv in runs:
            ops.attn_fwd(qkv, att, ctx, heads=2, lse=lse)
            ops.attn_bwd(qkv, att, ctx, dctx, lse, dqkv, heads=2)
        torch.cuda.synchronize()
        time.sleep(0.5)
    seq = []
    for ev in prof.events():
        nm = ev.name.replace(" ", "")
        nm = (nm[4:] if nm.startswith("void") else nm).split("(")[0].replace("hero::", "")
        if nm.startswith("attn_"):
            seq.append((ev.time_range.start, nm))
    return [nm for _, nm in sorted(seq)]


def test_every_case_launches_its_kernels():
    """Each dispatch case under the profiler: the forward and the backward launch exactly the
    kernels of the paths the plan contains, in order. The profiling runs in a child process of
    its own, so that this test's session is that process's first (see _kernel_sequence) and the
    profiler of the test process is left untouched for the tests that run after this one."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import json, sys; sys.path.insert(0, sys.argv[1]); "
            "from tests.test_attention_gpu import _kernel_sequence; "
            "print('KERNELS', json.dumps(_kernel_sequence()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code, root], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.split("KERNELS", 1)[1])
    want = []
    for lens in [lens for _, lens, _ in MATRIX] + [None]:
        fp, bp = _paths(_lens_plan(lens)[0] if lens is not None else _host_joint(_joint_with_long()))
        want += [FWD_KERNELS[p] for p in ("A1", "A2") if p in fp]
        want += [k for p in ("B1", "B2") if p in bp for k in BWD_KERNELS[p]]
    assert got == want, (got, want)


# ------------------------------------------------------------------------------ 2. exact probes
def _pos(hp):
    """Position of every token in its own sequence, and the sequence's length."""
    lo = np.asarray(hp["seq_lo"], np.int64)
    n = np.bincount(lo, minlength=hp["n_tok"])[lo]
    return np.arange(hp["n_tok"]) - lo, n


UNIFORM = [[1], [64], [65], [127], [128], [129], [768], [8] * 16, [1] * 16 + [5],
           [3, 64, 65, 129, 768, 127]]


@pytest.mark.parametrize("lens", UNIFORM, ids=["-".join(map(str, s[:4])) for s in UNIFORM])
def test_uniform_probe(lens):
    """Q = K = 0 and, at 12 heads, V of head h the one-hot of key position p - 64 h: ctx[i, 64 h +
    c] = 1/n for every key 64 h + c < n of the row's own sequence (up to the bf16 rounding of 1/n)
    and exactly 0 elsewhere; a lost key reads 0 where 1/n belongs. With uniform P the backward's
    dV_j is the mean of dO over the sequence."""
    heads = 12
    hp, att = _lens_plan(lens)
    n_tok, H = hp["n_tok"], heads * 64
    pos, n = _pos(hp)
    qkv = torch.zeros(n_tok, 3 * H, dtype=BF16, device=_dev())
    p = torch.as_tensor(pos, device=_dev())
    v = torch.zeros(n_tok, H, dtype=BF16, device=_dev())
    v[torch.arange(n_tok, device=_dev()), p] = 1          # column 64 h + c = key position
    qkv[:, 2 * H:] = v
    _, dctx = _inputs(hp, heads, seed=3)
    out, ref = _run(hp, att, heads, qkv, dctx, f"uniform {lens[:4]}")
    inv = torch.as_tensor(1.0 / n, device=_dev())[:, None]
    col = torch.arange(H, device=_dev())[None]
    own = col < torch.as_tensor(n, device=_dev())[:, None]
    ctx = out["ctx"].double()
    assert bool((ctx[~own.expand_as(ctx)] == 0).all()), "uniform probe: weight outside the sequence"
    want = inv.expand_as(ctx)[own.expand_as(ctx)]
    got = ctx[own.expand_as(ctx)]
    assert bool(((got - want).abs() <= _half_ulp(want) + 1e-4 * want).all()), "uniform probe: 1/n"
    # dV_j = mean_i dO_i over the sequence (the reference says so too)
    lo = torch.as_tensor(np.asarray(hp["seq_lo"], np.int64), device=_dev())
    mean = torch.zeros(n_tok, H, dtype=F64, device=_dev()).index_add_(0, lo, dctx.double())
    mean = mean[lo] * inv
    assert torch.allclose(ref["dqkv"][:, 2 * H:], mean, rtol=0, atol=1e-12)


NEEDLE = [[64], [65], [128], [7, 121], [129], [200], [768], [8] * 16]


@pytest.mark.parametrize("lens", NEEDLE, ids=["-".join(map(str, s[:4])) for s in NEEDLE])
def test_needle_probe(lens):
    """Key j(i) dominates row i by >= 20 scaled units, j(i) cycling through 0, 63, 64, 127 and n - 1:
    ctx_i equals v_j(i) exactly in bf16 (the other keys weigh < 768 e^-20 together)."""
    heads = 2
    hp, att = _lens_plan(lens)
    n_tok, H = hp["n_tok"], heads * 64
    pos, n = _pos(hp)
    lo = np.asarray(hp["seq_lo"], np.int64)
    gen = torch.Generator(device="cpu").manual_seed(len(lens) + n_tok)
    qkv = torch.randn(n_tok, 3 * H, generator=gen, dtype=F64)
    K = torch.where(torch.rand(n_tok, H, generator=gen) < 0.5, -1.0, 1.0).double()
    qkv[:, H:2 * H] = K
    targets = np.array([0, 63, 64, 127, -1])
    k = np.arange(n_tok) % len(targets)
    tgt = targets[k]
    tgt = np.where(tgt < 0, n - 1, tgt)
    tgt = np.where(tgt < n, tgt, n - 1)
    j = torch.as_tensor(lo + tgt)
    qkv[:, :H] = 5.0 * K[j]
    qkv = qkv.to(BF16).to(_dev())
    # the needle's margin, in scaled units, over every other key of the sequence and head
    q = qkv[:, :H].double().view(n_tok, heads, 64)
    kk = qkv[:, H:2 * H].double().view(n_tok, heads, 64)
    for s in np.unique(lo):
        rows = np.nonzero(lo == s)[0]
        sc = torch.einsum("ihd,jhd->hij", q[rows], kk[rows]) * SCALE
        top = sc.gather(2, torch.as_tensor(tgt[rows], device=_dev())[None, :, None].expand(heads, -1, 1))
        others = sc.masked_fill(sc == top, -math.inf).amax(-1, keepdim=True) if len(rows) > 1 else top - 99
        assert bool((top - others >= 20).all()), "needle margin"
    _, dctx = _inputs(hp, heads, seed=4)
    out, _ = _run(hp, att, heads, qkv, dctx, f"needle {lens[:4]}")
    assert torch.equal(out["ctx"], qkv[j.to(_dev()), 2 * H:]), "needle: ctx_i != v_j(i)"


# ------------------------------------------------------------------------------ 3. magnitudes
def _magnitude_qkv(kind, hp, heads, seed):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    n_tok, H = hp["n_tok"], heads * 64
    x = torch.randn(n_tok, 3 * H, generator=gen, dtype=F64)
    Q, K = x[:, :H].view(n_tok, heads, 64), x[:, H:2 * H].view(n_tok, heads, 64)
    if kind == "spread60":            # scaled scores spread over about +-60
        Q *= 4.0
        K *= 4.0
    elif kind == "offset960":         # every raw score 960 + a few units
        Q[..., 1:] *= 0.7
        K[..., 1:] *= 0.7
        Q[..., 0], K[..., 0] = 32.0, 30.0
    elif kind == "neighbours8000":    # even sequences' rows: odd sequences' keys 8000 raw above
        lo = np.asarray(hp["seq_lo"], np.int64)
        odd = torch.as_tensor(np.unique(lo, return_inverse=True)[1] % 2 == 1)
        Q[..., 0] = torch.where(odd, 0.0, 64.0)[:, None]
        K[..., 0] = torch.where(odd, 125.0, 0.0)[:, None]
    elif kind == "equal":             # every score of a row the same nonzero value
        Q.zero_()
        K.zero_()
        Q[..., 0], K[..., 0] = 10.0, 10.0
    return x.to(BF16).to(_dev())


MAGNITUDE = [("spread60", [37, 90, 1, 128, 200, 768]), ("offset960", [37, 90, 1, 128, 200, 768]),
             ("neighbours8000", [8] * 16 + [2, 5, 1, 7] * 6 + [60, 60]),
             ("equal", [37, 90, 1, 128, 200, 768])]


@pytest.mark.parametrize("kind,lens", MAGNITUDE, ids=[m[0] for m in MAGNITUDE])
def test_score_magnitudes(kind, lens):
    heads = 2
    hp, att = _lens_plan(lens)
    qkv = _magnitude_qkv(kind, hp, heads, seed=9)
    _, dctx = _inputs(hp, heads, seed=10)
    _run(hp, att, heads, qkv, dctx, f"magnitude {kind}")


# ------------------------------------------------------------------------------ 4-6
def test_writes_and_reads_stay_inside_n_tok():
    """Explicitly: a plan whose last tile ends at n_tok on each path, every output a row slice of a
    NaN buffer, NaN behind qkv and dctx (_run checks the same on every case)."""
    for lens in ([5, 60, 3], [300], [40, 130, 128]):
        hp, att = _lens_plan(lens)
        qkv, dctx = _inputs(hp, 12, seed=21)
        out = _launch(qkv, att, 12, dctx)
        _check_bytes(out, hp["n_tok"], 12, f"bytes {lens}")


def test_relaunch_is_bit_identical():
    heads = 12
    hp, att = _lens_plan([20, 200, 31, 129, 64, 100, 100, 9])
    qkv, dctx = _inputs(hp, heads, seed=31)
    a = _launch(qkv, att, heads, dctx)
    b = _launch(qkv, att, heads, dctx)
    for k in ("ctx", "lse", "dqkv"):
        assert torch.equal(a[k], b[k]), k
    # dbias accumulates with fp32 atomics: only its bound
    want = b["dbias0"] + b["dqkv"].double().sum(0)
    _within(b["dbias"], want, _dbias_tol(hp, b["dqkv"], b["dbias0"]), "relaunch dbias")


@pytest.mark.parametrize("lens", [[25, 90, 128, 7], [129, 768, 300]])
def test_backward_takes_the_header_lse(lens):
    """attn_bwd given the float64 reference lse (cast to fp32) instead of the forward's: the
    gradients stay within their bounds, so the forward and backward share the documented
    convention, not a private one."""
    heads = 2
    hp, att = _lens_plan(lens)
    qkv, dctx = _inputs(hp, heads, seed=41)
    ref = _reference(qkv, hp, heads)
    out = _launch(qkv, att, heads, dctx, lse_in=ref["lse"].float().contiguous())
    ref = _reference(qkv, hp, heads, dctx, out["ctx"])
    _check(out, ref, hp, heads, f"header lse {lens}")


# ------------------------------------------------------------------------------ 7. model plans
def _model_plans():
    from hero_b200 import synth
    from hero_b200.plan import build_plans, plan_inputs, qa_plan
    vb, qb = synth.syn_tvr_ragged(batch_size=6, vfeat_dim=8)
    rplan, _ = build_plans(plan_inputs(vb), plan_inputs(qb, "txt"))
    qa = synth.syn_videoqa_batch(n_videos=3, n_cand=3, vfeat_dim=8)
    return {"f_": lambda: _seq_plan(rplan.f.seq), "joint": lambda: _joint_case(rplan._joint),
            "c_": lambda: _seq_plan(rplan.c.seq), "qa": lambda: _seq_plan(qa_plan(qa).seq)}


@pytest.mark.parametrize("form", ["f_", "joint", "c_", "qa"])
def test_model_plan(form):
    hp, att = _model_plans()[form]()
    qkv, dctx = _inputs(hp, 12, seed=51)
    _run(hp, att, 12, qkv, dctx, f"model plan {form}")


def test_bench_scale_joint_plan():
    """The fused video + query pass of bench.py's batch (syn_tvr_dense, 32 clips)."""
    from hero_b200 import synth
    from hero_b200.plan import build_plans, plan_inputs
    vb, qb = synth.syn_tvr_dense(batch_size=32, vfeat_dim=8)
    rplan, _ = build_plans(plan_inputs(vb), plan_inputs(qb, "txt"))
    hp, att = _joint_case(rplan._joint)
    qkv, dctx = _inputs(hp, 12, seed=61)
    _run(hp, att, 12, qkv, dctx, "bench-scale joint plan")


# ------------------------------------------------------------------------------ 8. negative controls
@pytest.mark.parametrize("lens", [[25, 90, 7, 128], [300, 129]])
def test_negative_controls(lens):
    """Each check against a perturbed reference must fail: one key removed from one sequence (ctx
    and every gradient), lse shifted by 2^-6, two dbias columns swapped; on a long plan, the long
    bounds against a reference that rounds P to bf16 like the tile path (the tile bounds accept it)."""
    heads = 2
    H = heads * 64
    hp, att = _lens_plan(lens)
    qkv, dctx = _inputs(hp, heads, seed=71)
    out, ref = _run(hp, att, heads, qkv, dctx, f"controls {lens}")
    key = int(np.asarray(hp["tok0"])[0]) + 3
    bad = _reference(qkv, hp, heads, dctx, out["ctx"], drop_key=key)
    assert _n_bad(out["ctx"], bad["ctx"], _tol_bf16(bad["ctx"], bad["e_ctx"])) > 0
    for i in range(3):
        c = slice(i * H, (i + 1) * H)
        assert _n_bad(out["dqkv"][:, c], bad["dqkv"][:, c],
                      _tol_bf16(bad["dqkv"][:, c], bad["e_dqkv"][:, c])) > 0, i
    assert _n_bad(out["lse"], ref["lse"] + 2.0 ** -6, ref["tol_lse"]) > 0
    want = out["dbias0"] + out["dqkv"].double().sum(0)
    a, b = int(want.argmax()), int(want.argmin())
    swapped = want.clone()
    swapped[[a, b]] = want[[b, a]]
    assert _n_bad(out["dbias"], swapped, _dbias_tol(hp, out["dqkv"], out["dbias0"])) > 0
    if hp["n_long"]:
        rnd = _reference(qkv, hp, heads, dctx, out["ctx"], round_p=True)
        tile = _reference(qkv, hp, heads, dctx, out["ctx"], tile_bounds=True)
        emul = rnd["ctx"].to(BF16)
        assert _n_bad(emul, ref["ctx"], _tol_bf16(ref["ctx"], ref["e_ctx"])) > 0
        assert _n_bad(emul, tile["ctx"], _tol_bf16(tile["ctx"], tile["e_ctx"])) == 0
        dv = rnd["dqkv"][:, 2 * H:].to(BF16)
        assert _n_bad(dv, ref["dqkv"][:, 2 * H:], _tol_bf16(ref["dqkv"][:, 2 * H:],
                                                              ref["e_dqkv"][:, 2 * H:])) > 0
        assert _n_bad(dv, tile["dqkv"][:, 2 * H:], _tol_bf16(tile["dqkv"][:, 2 * H:],
                                                               tile["e_dqkv"][:, 2 * H:])) == 0


# ------------------------------------------------------------------------------ host checks
def test_attention_host_checks_raise_before_launch():
    """Arguments the kernels would read or write past their end, or misread, are refused on the
    host before any launch: the NaN-filled outputs stay NaN."""
    from hero_b200 import ops
    heads = 2
    H = heads * 64
    hp, att = _lens_plan([5, 60, 3])
    n = hp["n_tok"]
    qkv, dctx = _inputs(hp, heads, seed=81)
    ctx, lse, dqkv = _nan((n, H), BF16), _nan((n, heads), F32), _nan((n, 3 * H), BF16)
    fwd_bad = [dict(qkv=qkv[:n - 1]), dict(qkv=qkv[:, :3 * H - 64]), dict(qkv=qkv.float()),
               dict(ctx=ctx[:n - 1]), dict(ctx=ctx.float()), dict(ctx=_nan((n, H + 64), BF16)),
               dict(lse=lse[:n - 1]), dict(lse=lse.double()), dict(lse=_nan((heads, n), F32).t()),
               dict(att={**att, "tile_ntok": att["tile_ntok"].long()}),
               dict(att={**att, "tile_tok0": att["tile_tok0"][:-1]}),
               dict(att={**att, "seq_lo": att["seq_lo"][:n - 1]})]
    for kw in fwd_bad:
        a = dict(qkv=qkv, att=att, ctx=ctx, lse=lse)
        a.update(kw)
        with pytest.raises(ValueError, match="attn_fwd"):
            ops.attn_fwd(a["qkv"], a["att"], a["ctx"], heads=heads, lse=a["lse"])
    ok_ctx = torch.zeros(n, H, dtype=BF16, device=_dev())
    ok_lse = torch.zeros(n, heads, device=_dev())
    bwd_bad = [dict(qkv=qkv[:n - 1]), dict(ctx=ok_ctx[:n - 1]), dict(dctx=dctx.float()),
               dict(dctx=dctx[:n - 1]), dict(dqkv=dqkv[:n - 1]), dict(dqkv=dqkv.float()),
               dict(lse=None), dict(lse=ok_lse[:, :1]),
               dict(att={**att, "seq_hi": att["seq_hi"].long()})]
    for kw in bwd_bad:
        a = dict(qkv=qkv, att=att, ctx=ok_ctx, dctx=dctx, lse=ok_lse, dqkv=dqkv)
        a.update(kw)
        with pytest.raises(ValueError, match="attn_bwd"):
            ops.attn_bwd(a["qkv"], a["att"], a["ctx"], a["dctx"], a["lse"], a["dqkv"], heads=heads)
    torch.cuda.synchronize()
    for t in (ctx, lse, dqkv):
        assert bool(torch.isnan(t.float()).all())
