"""The row kernels of csrc/rowwise.cu against float64: every kernel that `hero_ln_fwd` /
`hero_ln_bwd` choose between, every LayerNorm call form of the model at its real width, and the
row utilities (colsum, cast, gather-sum, ReLU backward) at their edges.

Paths (the dispatch of hero_ln_fwd / hero_ln_bwd):
  F1 ln_fwd_fast_kernel<false>  h <= 768, bf16 x, no add_tab / add_vec / y_lo
  F2 ln_fwd_fast_kernel<true>   the same with fp32 x
  F3 ln_fwd_kernel<3, 1>        h <= 768 with a table / vector add or y_lo
  F4 ln_fwd_wide_kernel         h > 768, n_rows >= 64
  F5 ln_fwd_kernel<17, 1>       h > 768, n_rows < 64
  B1 / B2 ln_bwd_fast_kernel<bf16 / fp32 x>   row gradients of the fast form, no table gradients
  B3 ln_bwd_kernel<3, 1> + ln_param_grad_kernel    h <= 768 otherwise
  B4 ln_bwd_kernel<17, 1> + ln_param_grad_kernel   h > 768
  B5 ln_param_grad_kernel alone                    no row output (dgamma / dbeta only)
The grids of F1, B1 / B2, F4 and the h > 768 kernels are capped (2 112, 1 056 warps, 1 056 CTAs,
4 224 warps on 132 SMs) and persistent, with the next row prefetched: 5 000 rows run that loop.

The reference restates include/hero_b200.h (hero_ln_args) in float64 on the exact tensors the
kernel reads: s = X[x_rows] + add_tab[add_idx] + add_vec, biased variance, y = (s - mean) rstd
gamma + beta, times the dropout mask and scale, scattered to y_rows; the backward is autograd
through that expression (dx = d loss / d s, dx_drop = dx * mask2 * scale2, table gradients =
scatter-adds of dx without the *_pad_idx rows, dgamma, dbeta, dbias).

Dropout masks are read back from the kernels, never restated from the hash: with gamma = 0 and
beta = 1 the forward stores exactly keep * scale. The same read-back with the `drop2` parameters
gives the mask of dx_drop (every kernel indexes element (i, col) as i * h + col).
test_dropout_masks_agree_across_paths ties the paths' masks to each other and to the GEMM
epilogue's; every masked comparison also runs a negative control with the mask of the next row,
which must fail.

Tolerances, from the output types (u = 2^-24; "fp32 level" = 1e-5 relative, which covers the
~sqrt(k) u error of the fp32 sums of k <= 4352 terms with a wide margin):
  E      = 1e-5 (|xhat gamma| + |gamma| + |beta|) * keep * scale: the fp32 error of one output
           element before it is stored (xhat carries the fp32 error of mean and rstd);
  bf16 y = 2^-8 |ref| + 2 E  (round to nearest: |bf16(v) - v| <= 2^-8 |v|);
  y_f32  = 2 E;  y + y_lo = 2^-16 |ref| + 2 E  (the low half rounds v - bf16(v), <= 2^-8 |v|);
  mean   = 1e-5 mean_j |s_ij|;  rstd = 1e-5 rstd + the shift of a two-pass variance centred on
           the kernel's own mean: (mean - ref mean)^2 rstd^3 / 2;
  the kernel's mean error d_i = |mean_i - ref mean_i| moves xhat by e_i = d_i rstd_i; it is added
           to E as |gamma| e_i (this is what rows of offset 1e3 and spread 1e-2 exercise);
  dx     = 2^-8 |ref| + D, D = 2e-5 T + 2 P: T = rstd (|g dy| + |c1| + |xhat c2|) are the
           magnitudes of the fp32 terms of dx = rstd (g dy - c1 - xhat c2), and P = rstd e (|c2| +
           |xhat c1|) is what the mean error does to it (xhat moves by e, c2 by e c1);
  dgamma = 1e-4 sum_i |dy xhat| + 1e-5 sum_i |dy| + sum_i |dy| e_i, dbeta = 1e-4 sum_i |dy|
           (fp32 sums of unrounded fp32 terms: the bound is per column, so one wrong column
           cannot hide behind the largest one); table gradients = sum of (1e-4 T + D) over the
           rows scattered there;
  dbias  = the column sums of dx_drop (else dx). The fast backward sums the unrounded fp32 values
           (reference: float64 dx_drop, bound sum (1e-4 T + D)); ln_param_grad_kernel re-reads
           the stored bf16 rows (reference: the float64 sum of exactly those rows, bound 1e-4
           sum |.|). A backward on the fast kernels is B1 / B2 even after a y_lo forward (F3):
           y_lo is a forward output.
"""
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
NAN = float("nan")
REL32 = 1e-5
SUM32 = 1e-4

FWD_KERNELS = {"F1": "ln_fwd_fast_kernel<false>", "F2": "ln_fwd_fast_kernel<true>",
               "F3": "ln_fwd_kernel<3,1>", "F4": "ln_fwd_wide_kernel",
               "F5": "ln_fwd_kernel<17,1>"}
BWD_KERNELS = {"B1": {"ln_bwd_fast_kernel<false>"}, "B2": {"ln_bwd_fast_kernel<true>"},
               "B3": {"ln_bwd_kernel<3,1>", "ln_param_grad_kernel"},
               "B4": {"ln_bwd_kernel<17,1>", "ln_param_grad_kernel"},
               "B5": {"ln_param_grad_kernel"}}


def _dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _randn(shape, g, scale=1.0, dtype=F32):
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(dtype).to(_dev())


def _idx(vals):
    return torch.as_tensor(vals, dtype=torch.int32).to(_dev())


def _nan(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=_dev())


def _n_bad(got, ref, tol):
    """Elements outside |got - ref| <= tol (NaN counts as outside)."""
    err = (got.double() - ref.double()).abs()
    return int((~(err <= tol)).sum().item())


def _within(got, ref, tol, what):
    bad = _n_bad(got, ref, tol)
    if bad:
        err = (got.double() - ref.double()).abs()
        worst = int(torch.nan_to_num(err - tol, nan=float("inf")).argmax())
        raise AssertionError(f"{what}: {bad}/{err.numel()} out of tolerance; worst flat index "
                             f"{worst}: got {got.flatten()[worst].item():.6g}, ref "
                             f"{ref.flatten()[worst].item():.6g}, tol "
                             f"{tol.flatten()[worst].item():.3g}")


# ------------------------------------------------------------------------------ case building
def _case(*, h, n, seed, x_f32=False, x_tab=0, x_pad=None, add_tab=0, add_pad=None,
          add_vec=False, y_extra=None):
    """Inputs of one LayerNorm call. x_tab > 0: x is a table of that many rows gathered by x_rows
    (with repeats: several output rows read one feature row); add_tab > 0: a table added through
    add_idx; y_extra: y_rows scatter the n rows into a NaN buffer of n + y_extra rows. x_pad /
    add_pad: the index given to every 5th row (a padding row, which gets no table gradient)."""
    g = _gen(seed)
    c = {"h": h, "n": n}
    rows = x_tab if x_tab else n
    sc = torch.empty(rows, 1, dtype=F64).uniform_(0.5, 3.0, generator=g)
    off = torch.empty(rows, 1, dtype=F64).uniform_(-2.0, 2.0, generator=g)
    x = torch.randn(rows, h, generator=g, dtype=F64) * sc + off
    c["x"] = x.to(F32 if x_f32 else BF16).to(_dev())
    c["x_rows"] = None
    if x_tab:
        r = torch.randint(0, x_tab, (n,), generator=g)
        if n > 3:
            r[1::4] = r[0::4][:r[1::4].numel()]          # guaranteed duplicates
        if x_pad is not None:
            r[::5] = x_pad
        c["x_rows"] = _idx(r)
    c["x_pad"] = -1 if x_pad is None else x_pad
    c["add_tab"] = c["add_idx"] = None
    if add_tab:
        c["add_tab"] = _randn((add_tab, h), g, 0.5)
        a = torch.randint(0, add_tab, (n,), generator=g)
        if add_pad is not None:
            a[::5] = add_pad
        c["add_idx"] = _idx(a)
    c["add_pad"] = -1 if add_pad is None else add_pad
    c["add_vec"] = _randn((h,), g, 0.5) if add_vec else None
    c["gamma"] = _randn((h,), g)
    c["beta"] = _randn((h,), g, 0.5)
    c["ny"] = n if y_extra is None else n + y_extra
    c["y_rows"] = None if y_extra is None else _idx(torch.randperm(c["ny"], generator=g)[:n])
    c["dy"] = _randn((c["ny"], h), g, dtype=BF16)
    return c


def _gather_kw(c):
    return dict(x_rows=c["x_rows"], add_tab=c["add_tab"], add_idx=c["add_idx"],
                add_vec=c["add_vec"], y_rows=c["y_rows"])


def _fwd(c, eps, drop, *, y_f32=False, y_lo=False, gamma=None, beta=None):
    """ln_fwd on case c into NaN-filled buffers; returns (y, y_f32, y_lo, mean, rstd)."""
    from hero_b200 import ops
    n, h, ny = c["n"], c["h"], c["ny"]
    y = _nan((ny, h), BF16)
    yf = _nan((ny, h), F32) if y_f32 else None
    ylo = _nan((ny, h), BF16) if y_lo else None
    mean, rstd = _nan((n,), F32), _nan((n,), F32)
    ops.ln_fwd(c["x"], c["gamma"] if gamma is None else gamma,
               c["beta"] if beta is None else beta, eps, y, n_rows=n, mean=mean, rstd=rstd,
               drop=drop, y_f32=yf, y_lo=ylo, **_gather_kw(c))
    return y, yf, ylo, mean, rstd


def _read_mask(c, drop, **kw):
    """Keep mask [n, h] of the forward path that case c takes, read back with gamma = 0, beta = 1:
    every stored value is exactly keep * scale."""
    h = c["h"]
    y, yf, _, _, _ = _fwd(c, 1e-5, drop, gamma=torch.zeros(h, device=_dev()),
                          beta=torch.ones(h, device=_dev()), **kw)
    rows = c["y_rows"].long() if c["y_rows"] is not None else torch.arange(c["n"], device=_dev())
    y = y[rows].float()
    keep = y != 0
    assert torch.equal(y[keep], torch.full_like(y[keep], torch.tensor(drop[2]).to(BF16).item())), \
        "read-back mask values"
    if yf is not None:
        assert torch.equal(yf[rows][keep], torch.full_like(yf[rows][keep], drop[2]))
    return keep


def _wrong(mask):
    """Negative control: the mask of the next row (of the other half of the columns for one row)."""
    return mask.roll(1, 0) if mask.shape[0] > 1 else mask.roll(mask.shape[1] // 2, 1)


# ------------------------------------------------------------------------------ float64 reference
def _ref(c, eps, keep=None, scale=1.0, keep2=None, scale2=1.0, got_mean=None):
    """float64 forward and autograd backward of hero_ln_args on case c. Returns a dict with y,
    mean, rstd, dx, dx_drop, d_x_tab, d_add_tab, dgamma, dbeta and the tolerance terms."""
    n, h = c["n"], c["h"]
    X = c["x"].double().requires_grad_(True)
    s = X[c["x_rows"].long()] if c["x_rows"] is not None else X[:n]
    A = None
    if c["add_tab"] is not None:
        A = c["add_tab"].double().requires_grad_(True)
        s = s + A[c["add_idx"].long()]
    if c["add_vec"] is not None:
        s = s + c["add_vec"].double()
    s.retain_grad()
    G = c["gamma"].double().requires_grad_(True)
    B = c["beta"].double().requires_grad_(True)
    mean = s.mean(1, keepdim=True)
    var = ((s - mean) ** 2).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xhat = (s - mean) * rstd
    y = xhat * G + B
    m = torch.ones_like(y) if keep is None else keep.double() * scale
    y = y * m
    rows = c["y_rows"].long() if c["y_rows"] is not None else torch.arange(n, device=_dev())
    dyr = c["dy"].double()[rows]
    (y * dyr).sum().backward()
    r = {"y": y.detach(), "mean": mean.detach().squeeze(1), "rstd": rstd.detach().squeeze(1),
         "dx": s.grad, "dgamma": G.grad, "dbeta": B.grad, "rows": rows}
    m2 = torch.ones_like(y) if keep2 is None else keep2.double() * scale2
    r["dx_drop"] = s.grad * m2
    r["d_x_tab"] = None if c["x_rows"] is None else X.grad.clone()
    if r["d_x_tab"] is not None and c["x_pad"] >= 0:
        r["d_x_tab"][c["x_pad"]] = 0
    r["d_add_tab"] = None if A is None else A.grad.clone()
    if A is not None and c["add_pad"] >= 0:
        r["d_add_tab"][c["add_pad"]] = 0
    # tolerance terms
    xh, gam = xhat.detach(), G.detach()
    rs = r["rstd"][:, None]
    e = torch.zeros_like(rs)
    if got_mean is not None:
        e = (got_mean.double() - r["mean"]).abs()[:, None] * rs
    r["e"] = e
    r["E"] = REL32 * ((xh * gam).abs() + gam.abs() + B.detach().abs()) * m + gam.abs() * e * m
    d = dyr * m                          # the gradient that reaches the LayerNorm output
    gy = d * gam
    c1 = gy.mean(1, keepdim=True)
    c2 = (gy * xh).mean(1, keepdim=True)
    r["T"] = rs * (gy.abs() + c1.abs() + (xh * c2).abs())
    # a kernel mean off by d shifts its xhat by e and its c2 by e c1: dx moves by
    # rstd e (c2 + xhat c1)
    r["P"] = rs * e * (c2.abs() + (xh * c1).abs())
    r["m2"] = m2
    r["d"] = d
    r["xhat"] = xh
    r["abs_s_mean"] = s.detach().abs().mean(1)
    return r


# ------------------------------------------------------------------------------ bounds
def _tol_y(r):
    return 2 ** -8 * r["y"].abs() + 2 * r["E"]


def _tol_dx(r, key="dx"):
    """bf16 dx (key "dx") or dx_drop (key "dx_drop": the same bound through mask2 * scale2)."""
    m = r["m2"] if key == "dx_drop" else 1.0
    return 2 ** -8 * r[key].abs() + (2 * REL32 * r["T"] + 2 * r["P"]) * m


def _tol_dgamma(r):
    d = r["d"]
    return (SUM32 * (d * r["xhat"]).abs().sum(0) + REL32 * d.abs().sum(0) +
            (d.abs() * r["e"]).sum(0))


# ------------------------------------------------------------------------------ one full case
def _check_fwd(c, r, y, yf, ylo, mean, rstd, what):
    rows = r["rows"]
    _within(mean, r["mean"], REL32 * r["abs_s_mean"], f"{what} mean")
    dm = (mean.double() - r["mean"]).abs()
    _within(rstd, r["rstd"], r["rstd"] * (REL32 + 0.5 * dm ** 2 * r["rstd"] ** 2), f"{what} rstd")
    _within(y[rows], r["y"], _tol_y(r), f"{what} y")
    unwritten = torch.ones(c["ny"], dtype=torch.bool, device=_dev())
    unwritten[rows] = False
    assert bool(torch.isnan(y[unwritten].float()).all()), f"{what}: a row outside y_rows written"
    if yf is not None:
        _within(yf[rows], r["y"], 2 * r["E"], f"{what} y_f32")
        assert bool(torch.isnan(yf[unwritten]).all()), f"{what}: y_f32 outside y_rows written"
    if ylo is not None:
        _within(y[rows].double() + ylo[rows].double(), r["y"], 2 ** -16 * r["y"].abs() + 2 * r["E"],
                f"{what} y + y_lo")
        assert bool(torch.isnan(ylo[unwritten].float()).all()), f"{what}: y_lo outside y_rows"


def _bwd(c, mean, rstd, drop, *, dx=True, dx_drop=None, d_x_tab=False, d_add_tab=False,
         dgb=True, dbias=False):
    """ln_bwd on case c; returns the outputs that were asked for (gradients start at zero)."""
    from hero_b200 import ops
    n, h = c["n"], c["h"]
    o = {"dx": _nan((n, h), BF16) if dx else None,
         "dx_drop": _nan((n, h), BF16) if dx_drop is not None else None,
         "d_x_tab": torch.zeros_like(c["x"], dtype=F32) if d_x_tab else None,
         "d_add_tab": torch.zeros_like(c["add_tab"]) if d_add_tab else None,
         "dgamma": torch.zeros(h, device=_dev()) if dgb else None,
         "dbeta": torch.zeros(h, device=_dev()) if dgb else None,
         "dbias": torch.zeros(h, device=_dev()) if dbias else None}
    ops.ln_bwd(c["dy"], c["x"], c["gamma"], mean, rstd, n_rows=n, drop=drop,
               drop2=dx_drop if dx_drop is not None else (0, 0, 1.0), x_pad_idx=c["x_pad"],
               add_pad_idx=c["add_pad"], **_gather_kw(c), **o)
    return o


def _check_bwd(c, r, o, fast, what):
    T, D = r["T"], 2 * REL32 * r["T"] + 2 * r["P"]      # D: the fp32 error of one dx element
    for k in ("dx", "dx_drop"):
        if o[k] is not None:
            _within(o[k], r[k], _tol_dx(r, k), f"{what} {k}")
    if o["dgamma"] is not None:
        _within(o["dgamma"], r["dgamma"], _tol_dgamma(r), f"{what} dgamma")
        _within(o["dbeta"], r["dbeta"], SUM32 * r["d"].abs().sum(0), f"{what} dbeta")
    if o["dbias"] is not None:
        if fast:       # unrounded fp32 dx_drop (dx) summed in registers
            src = r["dx_drop"] if o["dx_drop"] is not None else r["dx"]
            _within(o["dbias"], src.sum(0), ((SUM32 * T + D) * r["m2"]).sum(0), f"{what} dbias")
        else:          # ln_param_grad_kernel re-reads the stored bf16 rows
            src = (o["dx_drop"] if o["dx_drop"] is not None else o["dx"]).double()
            _within(o["dbias"], src.sum(0), SUM32 * src.abs().sum(0), f"{what} dbias")
    for k, idx, pad in (("d_x_tab", c["x_rows"], c["x_pad"]),
                        ("d_add_tab", c["add_idx"], c["add_pad"])):
        if o[k] is None:
            continue
        tol = torch.zeros_like(r[k]).index_add_(0, idx.long(), SUM32 * T + D)
        _within(o[k], r[k], tol, f"{what} {k}")
        if pad >= 0:
            assert bool((o[k][pad] == 0).all()), f"{what}: {k} wrote its padding row {pad}"


def _run(c, eps, *, p=0.0, p2=0.0, y_f32=False, y_lo=False, bwd=None, fast_bwd=False,
         what="", key=0x5EED):
    """Forward (checked), then the backward with the outputs in `bwd` (checked), both against the
    float64 reference under the read-back masks, with a wrong-mask negative control."""
    from hero_b200 import ops
    drop = ops.drop_params(p, key)
    drop2 = ops.drop_params(p2, key ^ 0xA5A5) if p2 else None
    y, yf, ylo, mean, rstd = _fwd(c, eps, drop, y_f32=y_f32, y_lo=y_lo)
    keep = _read_mask(c, drop, y_f32=y_f32, y_lo=y_lo) if p else None
    keep2 = None
    if p2:    # mask of the dx_drop copy: the same read-back under the drop2 parameters
        keep2 = _read_mask(c, drop2, y_f32=y_f32, y_lo=y_lo)
    r = _ref(c, eps, keep, drop[2], keep2, drop2[2] if p2 else 1.0, got_mean=mean)
    _check_fwd(c, r, y, yf, ylo, mean, rstd, what)
    o = None
    if bwd is not None:
        o = _bwd(c, mean, rstd, drop, dx_drop=drop2, **bwd)
        _check_bwd(c, r, o, fast_bwd, what)
    if p:     # negative controls: the next row's mask must fail the same comparisons
        rw = _ref(c, eps, _wrong(keep), drop[2], keep2, drop2[2] if p2 else 1.0, got_mean=mean)
        assert _n_bad(y[rw["rows"]], rw["y"], _tol_y(rw)) > 0, \
            f"{what}: forward negative control passed"
        if o is not None:
            bad = 0
            if o["dx"] is not None:
                bad += _n_bad(o["dx"], rw["dx"], _tol_dx(rw))
            if o["dgamma"] is not None:
                bad += _n_bad(o["dgamma"], rw["dgamma"], _tol_dgamma(rw))
            assert bad > 0, f"{what}: backward negative control passed"
    if p2 and o is not None and o["dx_drop"] is not None:
        rw = _ref(c, eps, keep, drop[2], _wrong(keep2), drop2[2], got_mean=mean)
        assert _n_bad(o["dx_drop"], rw["dx_drop"], _tol_dx(rw, "dx_drop")) > 0, \
            f"{what}: dx_drop negative control passed"
    return r


# ------------------------------------------------------------------------------ dispatch matrix
ROWS_GRAD = dict(dx=True, dgb=True)
# (id, forward path, backward path, case kwargs, eps, p, p2, run kwargs)
MATRIX = [
    # F1 / B1: bf16 rows of <= 768, gathered and scattered rows on the fast kernels too
    ("F1-B1-h8-n1", dict(h=8, n=1), 1e-12, 0.0, 0.0, dict(bwd=ROWS_GRAD)),
    ("F1-B1-h136-n65-rows", dict(h=136, n=65, x_tab=40, y_extra=30), 1e-5, 0.1, 0.0,
     dict(bwd=dict(dx=True, dgb=True, dbias=True))),
    ("F1-B1-h768-n5000-rows-drop2", dict(h=768, n=5000, x_tab=3000, y_extra=77), 1e-12, 0.1, 0.1,
     dict(bwd=dict(dx=True, dgb=True, dbias=True))),
    # F2 / B2: fp32 rows (the residual stream), TVC decode-step row counts
    ("F2-B2-h768-n3", dict(h=768, n=3, x_f32=True), 1e-12, 0.0, 0.0,
     dict(y_f32=True, bwd=ROWS_GRAD)),
    ("F2-B2-h8-n63", dict(h=8, n=63, x_f32=True, y_extra=5), 1e-5, 0.1, 0.1,
     dict(y_f32=True, bwd=dict(dx=False, dgb=True, dbias=True))),
    ("F2-B2-h136-n5000-drop2", dict(h=136, n=5000, x_f32=True), 1e-12, 0.1, 0.1,
     dict(y_f32=True, bwd=dict(dx=True, dgb=True, dbias=True))),
    # F3 / B3: adds, y_lo, table gradients with padding rows
    ("F3-B3-h8-n64-vec", dict(h=8, n=64, add_vec=True), 1e-5, 0.1, 0.0,
     dict(y_f32=True, bwd=ROWS_GRAD)),
    ("F3-B3-h136-n5000-tables", dict(h=136, n=5000, x_f32=True, x_tab=700, x_pad=1, add_tab=50,
                                     add_pad=0, add_vec=True, y_extra=100), 1e-12, 0.1, 0.1,
     dict(y_f32=True, bwd=dict(dx=True, d_x_tab=True, d_add_tab=True, dgb=True, dbias=True))),
    ("F3-B1-h768-n1-ylo", dict(h=768, n=1), 1e-5, 0.0, 0.0,
     dict(y_lo=True, bwd=dict(dx=True, dgb=True, dbias=True))),
    ("F3-B3-h768-n3-tab", dict(h=768, n=3, x_tab=2, x_pad=0, add_tab=4), 1e-12, 0.1, 0.0,
     dict(bwd=dict(dx=False, d_x_tab=True, dgb=True))),
    # F4 / B4 + B5: wide rows, at and above the switch, and beyond every grid cap
    ("F4-B4-h776-n64", dict(h=776, n=64, y_extra=3), 1e-12, 0.1, 0.1,
     dict(bwd=dict(dx=True, dgb=True, dbias=True))),
    ("F4-B4-h2048-n65-tables", dict(h=2048, n=65, x_f32=True, x_tab=20, x_pad=3, add_tab=3,
                                    add_pad=0), 1e-5, 0.0, 0.0,
     dict(bwd=dict(dx=True, d_x_tab=True, d_add_tab=True, dgb=True))),
    ("F4-B4-h4352-n5000-ylo", dict(h=4352, n=5000, x_f32=True, x_tab=1200, add_tab=2,
                                   add_pad=0), 1e-5, 0.1, 0.0,
     dict(y_lo=True, bwd=dict(dx=False, d_add_tab=True, dgb=True))),
    # F5 / B4 + B5: wide rows below the switch
    ("F5-B4-h776-n63", dict(h=776, n=63, x_tab=30, y_extra=9), 1e-5, 0.1, 0.1,
     dict(y_lo=True, bwd=dict(dx=True, dgb=True, dbias=True))),
    ("F5-B4-h2048-n3-tables", dict(h=2048, n=3, x_f32=True, x_tab=2, add_tab=2, add_pad=1,
                                   add_vec=True), 1e-12, 0.1, 0.0,
     dict(bwd=dict(dx=True, d_add_tab=True, dgb=True))),
    ("F5-B4-h4352-n1", dict(h=4352, n=1, x_f32=True), 1e-12, 0.0, 0.0, dict(bwd=ROWS_GRAD)),
    # B5 alone (dgamma / dbeta, no row output)
    ("F1-B5-h136-n5000", dict(h=136, n=5000), 1e-5, 0.0, 0.0, dict(bwd=dict(dx=False))),
    ("F5-B5-h4352-n63", dict(h=4352, n=63, x_f32=True, x_tab=21), 1e-5, 0.1, 0.0,
     dict(y_lo=True, bwd=dict(dx=False))),
]


@pytest.mark.parametrize("name,ckw,eps,p,p2,kw", MATRIX, ids=[m[0] for m in MATRIX])
def test_ln_dispatch_matrix(name, ckw, eps, p, p2, kw):
    fast = name.split("-")[1] in ("B1", "B2")
    c = _case(seed=zlib.crc32(name.encode()) & 0xFFFF, **ckw)
    _run(c, eps, p=p, p2=p2, fast_bwd=fast, what=name, **kw)


# ------------------------------------------------------------------------------ masks
def test_dropout_masks_agree_across_paths():
    """F1 / F2 / F3 give one mask per (key, i, h) (element index i * h + col, whatever y_rows is),
    F4 and F5 likewise, and at h = 768 it is the GEMM epilogue's mask. Negative control: another
    key's mask differs."""
    from hero_b200 import ops
    from tests.test_dropout_parity_gpu import _elementwise_mask
    drop = ops.drop_params(0.1, 0xD00D)
    for h in (8, 136, 768):
        n = 5000
        base = _read_mask(_case(h=h, n=n, seed=1), drop)                           # F1
        assert abs(base.float().mean().item() - 0.9) < 0.02
        assert torch.equal(_read_mask(_case(h=h, n=n, seed=2, y_extra=11), drop), base)  # F1 rows
        assert torch.equal(_read_mask(_case(h=h, n=n, seed=3, x_f32=True), drop), base)  # F2
        assert torch.equal(_read_mask(_case(h=h, n=n, seed=4, add_vec=True, y_extra=5), drop),
                           base)                                                   # F3
        assert torch.equal(_read_mask(_case(h=h, n=n, seed=5), drop, y_lo=True), base)  # F3 y_lo
        other = _read_mask(_case(h=h, n=n, seed=1), ops.drop_params(0.1, 0xD00E))
        assert not torch.equal(other, base)
        if h == 768:
            assert torch.equal(_elementwise_mask(n, h, drop), base)
    for h in (776, 2048, 4352):
        wide = _read_mask(_case(h=h, n=200, seed=6, x_f32=True), drop)             # F4
        assert torch.equal(_read_mask(_case(h=h, n=200, seed=7, y_extra=13), drop), wide)
        for n in (1, 63):                                                           # F5
            assert torch.equal(_read_mask(_case(h=h, n=n, seed=8, x_f32=True), drop), wide[:n])
            assert torch.equal(_read_mask(_case(h=h, n=n, seed=9, y_extra=4, add_vec=True), drop),
                               wide[:n])


def test_every_dispatch_cell_runs_its_kernel():
    """One small case per cell under the profiler: the kernels that ran are the cell's."""
    from torch.profiler import ProfilerActivity, profile

    from hero_b200 import ops
    cells = [  # (forward path, backward path, case kwargs, forward kwargs, backward kwargs)
        ("F1", "B1", dict(h=136, n=3), {}, ROWS_GRAD),
        ("F2", "B2", dict(h=768, n=5, x_f32=True), dict(y_f32=True), ROWS_GRAD),
        ("F3", "B3", dict(h=8, n=64, add_vec=True), {}, ROWS_GRAD),
        ("F3", "B3", dict(h=768, n=3, x_tab=4), dict(y_lo=True), dict(dx=False, d_x_tab=True)),
        ("F4", "B4", dict(h=776, n=64), {}, ROWS_GRAD),
        ("F5", "B4", dict(h=4352, n=63, x_f32=True, add_tab=2), {},
         dict(dx=False, d_add_tab=True, dgb=True)),
        ("F5", "B5", dict(h=776, n=1), {}, dict(dx=False)),
        ("F1", "B5", dict(h=768, n=63), {}, dict(dx=False)),
    ]
    ln = {"ln_fwd", "ln_bwd", "ln_param"}
    for fp, bp, ckw, fkw, bkw in cells:
        c = _case(seed=3, **ckw)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, _, _, mean, rstd = _fwd(c, 1e-5, ops.drop_params(0.1, 5), **fkw)
            torch.cuda.synchronize()
        ran_f = _ln_kernels(prof, ln)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _bwd(c, mean, rstd, ops.drop_params(0.1, 5), **bkw)
            torch.cuda.synchronize()
        ran_b = _ln_kernels(prof, ln)
        assert ran_f == {FWD_KERNELS[fp]}, (fp, ckw, ran_f)
        assert ran_b == BWD_KERNELS[bp], (bp, ckw, ran_b)


def _ln_kernels(prof, prefixes):
    names = set()
    for ev in prof.events():
        nm = ev.name.replace(" ", "")
        if nm.startswith("void"):
            nm = nm[4:]
        nm = nm.split("(")[0].replace("hero::", "")
        if any(nm.startswith(p) for p in prefixes):
            names.add(nm)
    return names


# ------------------------------------------------------------------------------ model call forms
def _txt_case(n, seed):
    """Text tokens: word table rows (pad id 1 on some tokens, ids repeated), position rows, the
    type row, scattered into the packed token rows of a larger NaN buffer."""
    return _case(h=768, n=n, seed=seed, x_f32=True, x_tab=1000, x_pad=1, add_tab=514,
                 add_vec=True, y_extra=n // 3 + 1)


@pytest.mark.parametrize("n", [5, 1500])
def test_form_text_embedding(n):
    """functional.py _txt_seg_fwd / _txt_seg_bwd: dropout, y_f32, d_x_tab with the pad row."""
    _run(_txt_case(n, 100 + n), 1e-5, p=0.1, y_f32=True,
         bwd=dict(dx=True, d_x_tab=True, dgb=True), what="text embedding")


@pytest.mark.parametrize("n", [7, 2300])
def test_form_frame_embedding(n):
    """functional.py _frame_seg_fwd / _frame_seg_bwd: bf16 frames + pos[t], scattered tokens."""
    c = _case(h=768, n=n, seed=200 + n, add_tab=100, y_extra=n // 2)
    _run(c, 1e-5, p=0.1, y_f32=True, bwd=dict(dx=True, dgb=True), what="frame embedding")


@pytest.mark.parametrize("n", [40, 63, 64, 300])
def test_form_image_layernorm(n):
    """functional.py:312 / 374: fp32 4352-wide features gathered (several tokens per feature row)
    with mask_emb[img_mask] added; the backward writes d_add_tab (pad row 0) and dgamma / dbeta."""
    c = _case(h=4352, n=n, seed=300 + n, x_f32=True, x_tab=max(2, n // 3), add_tab=2, add_pad=0)
    _run(c, 1e-5, bwd=dict(dx=False, d_add_tab=True, dgb=True), what="image LN")


@pytest.mark.parametrize("n", [9, 700])
def test_form_image_output_layernorm(n):
    """functional.py:320 / 353: bf16 projection + img pos rows + type row, dropout, y_f32."""
    c = _case(h=768, n=n, seed=400 + n, add_tab=100, add_vec=True, y_extra=n)
    _run(c, 1e-5, p=0.1, y_f32=True, bwd=dict(dx=True, dgb=True), what="image output LN")


@pytest.mark.parametrize("n", [12, 63, 64, 900])
def test_form_frame_transform_layernorm(n):
    """functional.py:403 / 442: gathered fp32 frame features, dropout, y_lo; backward dgamma /
    dbeta only (path B5)."""
    c = _case(h=4352, n=n, seed=500 + n, x_f32=True, x_tab=max(2, n // 4))
    _run(c, 1e-5, p=0.1, y_lo=True, bwd=dict(dx=False, dgb=True), what="frame_transform LN")


@pytest.mark.parametrize("n", [1, 3200])
def test_form_transformer_layer(n):
    """csrc/stack.cu: fp32 pre-LN sum, y + y_f32; backward dx, dx_drop under drop2, dgamma /
    dbeta and dbias (the bias gradient of the Linear feeding the LayerNorm)."""
    c = _case(h=768, n=n, seed=600 + n, x_f32=True)
    _run(c, 1e-12, p2=0.1, y_f32=True, fast_bwd=True,
         bwd=dict(dx=True, dgb=True, dbias=True), what="transformer layer LN")


@pytest.mark.parametrize("n", [1, 4, 80])
def test_form_tvc_decode_step(n):
    """tvc.py _positions: the embedding LN (word rows + position rows, y_f32), the layer LNs on
    the fp32 sum (y_f32) and the LM-head LN on bf16 rows, on the rows of one decode step, into
    buffers sized for more rows (rows past n_rows stay untouched)."""
    from hero_b200 import ops
    emb = _case(h=768, n=n, seed=701 + n, x_f32=True, x_tab=300, add_tab=100)
    _run(emb, 1e-5, y_f32=True, what="tvc embedding LN")
    m = n + 16
    for x_f32, y_f32, eps in ((True, True, 1e-12), (False, False, 1e-12)):
        c = _case(h=768, n=n, seed=702 + n + x_f32, x_f32=x_f32)
        y, yf = _nan((m, 768), BF16), (_nan((m, 768), F32) if y_f32 else None)
        ops.ln_fwd(c["x"], c["gamma"], c["beta"], eps, y, n_rows=n, y_f32=yf)
        r = _ref(c, eps)
        _within(y[:n], r["y"], _tol_y(r), "tvc LN y")
        assert bool(torch.isnan(y[n:].float()).all())
        if yf is not None:
            _within(yf[:n], r["y"], 2 * r["E"], "tvc LN y_f32")
            assert bool(torch.isnan(yf[n:]).all())


# ------------------------------------------------------------------------------ edge rows
@pytest.mark.parametrize("h,n", [(768, 200), (136, 5000), (4352, 40), (4352, 100)])
def test_large_offset_zero_and_outlier_rows(h, n):
    """Rows of offset 1e3 and spread 1e-2 (a one-pass E[x^2] - mean^2 variance loses every digit
    there), all-zero rows, and a row 1e4 times larger beside small ones; fp32 x on the fast path
    (h <= 768, also through a vector add: path F3) and both wide paths."""
    g = _gen(800 + h + n)
    x = torch.randn(n, h, generator=g, dtype=F64) * 1e-2 + 1e3
    x[1::7] = 0
    x[2::7] = torch.randn(h, generator=g, dtype=F64) * 1e-3
    x[3::7] = torch.randn(h, generator=g, dtype=F64) * 1e4
    x[4::7] = torch.randn(h, generator=g, dtype=F64) * 1e-3 - 5.0
    for add_vec in ((False, True) if h <= 768 else (False,)):
        c = _case(h=h, n=n, seed=801, x_f32=True, add_vec=add_vec)
        c["x"] = x.to(F32).to(_dev())
        if add_vec:
            c["add_vec"] = torch.zeros(h, device=_dev())
        for eps in (1e-12, 1e-5):
            r = _run(c, eps, bwd=dict(dx=True, dgb=True), fast_bwd=not add_vec and h <= 768,
                     what=f"edge rows h={h} add_vec={add_vec} eps={eps}")
            zero = r["rstd"][1::7]
            assert torch.allclose(zero, torch.full_like(zero, eps ** -0.5))


# ------------------------------------------------------------------------------ host checks
def test_ln_host_checks_raise_before_launch():
    """An int64 y_rows and per-row tensors shorter than n_rows are refused before any launch:
    the NaN-filled outputs stay NaN."""
    from hero_b200 import ops
    n, h = 6, 16
    x = torch.zeros(n, h, dtype=BF16, device=_dev())
    gamma, beta = torch.ones(h, device=_dev()), torch.zeros(h, device=_dev())
    mean, rstd = torch.zeros(n, device=_dev()), torch.ones(n, device=_dev())
    rows32 = torch.arange(n, dtype=torch.int32, device=_dev())
    short = torch.zeros(n - 1, device=_dev())
    y = _nan((n, h), BF16)
    fwd_bad = [dict(y_rows=rows32.long()), dict(mean=short), dict(rstd=short),
               dict(y_rows=rows32[:n - 1]), dict(x_rows=rows32[:n - 1]),
               dict(add_tab=torch.zeros(2, h, device=_dev()), add_idx=rows32[:n - 1] * 0)]
    for kw in fwd_bad:
        args = dict(mean=_nan((n,), F32), rstd=_nan((n,), F32))
        args.update(kw)
        with pytest.raises(ValueError, match="ln_fwd"):
            ops.ln_fwd(x, gamma, beta, 1e-5, y, n_rows=n, **args)
    with pytest.raises(ValueError, match="ln_fwd"):
        ops.ln_fwd(x, gamma, beta, 1e-5, y[:n - 1], n_rows=n)
    with pytest.raises(ValueError, match="ln_fwd"):
        ops.ln_fwd(x[:n - 1], gamma, beta, 1e-5, y, n_rows=n)
    torch.cuda.synchronize()
    assert bool(torch.isnan(y.float()).all())
    dy = torch.ones(n, h, dtype=BF16, device=_dev())
    dx = _nan((n, h), BF16)
    bwd_bad = [dict(y_rows=rows32.long()), dict(mean=short), dict(rstd=short),
               dict(dy=dy[:n - 1]), dict(dx=dx[:n - 1]), dict(dx_drop=dx[:n - 1], dx=None)]
    for kw in bwd_bad:
        args = dict(dy=dy, mean=mean, rstd=rstd, dx=dx)
        args.update(kw)
        with pytest.raises(ValueError, match="ln_bwd"):
            ops.ln_bwd(args.pop("dy"), x, gamma, args.pop("mean"), args.pop("rstd"), n_rows=n,
                       **args)
    torch.cuda.synchronize()
    assert bool(torch.isnan(dx.float()).all())


# ------------------------------------------------------------------------------ row utilities
@pytest.mark.parametrize("m", [1, 7, 9, 33])
@pytest.mark.parametrize("n", [8, 264])
def test_colsum_strided_rows(m, n):
    """out += column sums of x[:, :n] inside rows of ld = n + 16 whose tail is NaN."""
    from hero_b200 import ops
    g = _gen(900 + m * n)
    full = torch.full((m, n + 16), NAN, dtype=BF16)
    full[:, :n] = torch.randn(m, n, generator=g).to(BF16)
    full = full.to(_dev())
    x = full[:, :n]
    assert x.stride(0) == n + 16
    out0 = _randn((n,), g)
    out = out0.clone()
    ops.colsum(x, out)
    ref = out0.double() + x.double().sum(0)
    _within(out, ref, SUM32 * (x.double().abs().sum(0) + out0.double().abs()), "colsum")


@pytest.mark.parametrize("n", [1, 5, 7, 9, 15, 1003])
def test_cast_bf16_tail(n):
    """The tail loop of cast_kernel (n % 8 != 0, n < 8): bit-exact round-to-nearest-even, with
    nothing written past n."""
    from hero_b200 import ops
    g = _gen(1000 + n)
    src = torch.randn(n, generator=g) * 10.0 ** torch.randint(-30, 30, (n,), generator=g)
    src[::3] = torch.tensor([1.0 + 2 ** -8, -(1.0 + 3 * 2 ** -8), float("inf")])[
        torch.arange(0, n, 3) % 3]
    src = src.to(_dev())
    buf = _nan((n + 16,), BF16)
    ops.cast_bf16(src, buf[:n])
    assert torch.equal(buf[:n].view(torch.int16), src.to(BF16).view(torch.int16))
    assert bool(torch.isnan(buf[n:].float()).all())


@pytest.mark.parametrize("h", [8, 4352])
def test_gather_sum_rows_empty_and_long_lists(h):
    """bf16 (overwrite) and fp32 (accumulate) gather-sums with empty lists, and for the fp32
    kernel lists longer than its 64 blocks x 32 entries (2 049, 5 000), which loop."""
    from hero_b200 import ops
    g = _gen(1100 + h)
    src = _randn((600, h), g, dtype=BF16)
    counts = torch.tensor([0, 3, 0, 1, 2049, 0, 5000, 2, 0])
    off = _idx(torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]))
    idx = _idx(torch.randint(0, 600, (int(counts.sum()),), generator=g))
    rows = torch.repeat_interleave(torch.arange(counts.numel()), counts).to(_dev())
    terms = src.double()[idx.long()]
    ref = torch.zeros(counts.numel(), h, dtype=F64, device=_dev()).index_add_(0, rows, terms)
    mag = torch.zeros_like(ref).index_add_(0, rows, terms.abs())
    short = counts <= 3
    sel = short.nonzero().squeeze(1)
    s_off = _idx(torch.cat([torch.zeros(1, dtype=torch.long), counts[short].cumsum(0)]))
    s_idx = torch.cat([idx[int(off[i]):int(off[i + 1])] for i in sel.tolist()])
    out = _nan((sel.numel(), h), BF16)
    ops.gather_sum_rows(src, s_off, s_idx, out)
    _within(out, ref[sel.to(_dev())], 2 ** -8 * ref[sel.to(_dev())].abs() +
            2 * SUM32 * mag[sel.to(_dev())], "gather_sum bf16")
    empty = (counts[short] == 0).nonzero().squeeze(1).to(_dev())
    assert bool((out[empty] == 0).all())
    base = _randn((counts.numel(), h), g)
    acc = base.clone()
    ops.gather_sum_rows(src, off, idx, acc)
    _within(acc, base.double() + ref, SUM32 * (mag + base.double().abs()), "gather_sum f32")
    assert torch.equal(acc[(counts == 0).to(_dev())], base[(counts == 0).to(_dev())])


def test_relu_bwd_signed_zero():
    """out = dy where pre > 0, else +0: pre = +0 and -0 both block the gradient; the smallest
    positive bf16 passes it."""
    from hero_b200 import ops
    g = _gen(1200)
    n = 8 * 131
    pre = torch.randn(n, generator=g).to(BF16)
    pre[0::4] = 0.0
    pre[1::4] = -0.0
    pre[2::8] = torch.tensor(1e-40).to(BF16)           # subnormal, > 0
    dy = torch.randn(n, generator=g).to(BF16)
    pre, dy = pre.to(_dev()), dy.to(_dev())
    assert bool(torch.signbit(pre[1::4].float()).all())
    out = _nan((n,), BF16)
    ops.relu_bwd(dy, pre, out)
    want = torch.where(pre.float() > 0, dy, torch.zeros_like(dy))
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    assert bool((out[0::4] == 0).all() and (out[1::4] == 0).all())
    assert torch.equal(out[2::8], dy[2::8])
