"""TEST INFRASTRUCTURE: torch restatement of the segment-table optimizer entry points
(include/hero_b200.h: hero_adamw_step_groups / hero_sumsq_segments_f32), so FusedAdamW with
parameter groups runs on a CPU-only box. A grouped step is the single-range restatement of
tests/fake_ops.py applied to each segment with its group's values, which is the contract the GPU
kernel is checked against bitwise."""
from tests import fake_ops


def adamw_step_groups(p, g, m, v, p_bf16, table, *, step_sizes, lr_wds, beta1, beta2, eps,
                      grad_scale=1.0, clip_sumsq=None, clip_max_norm=0.0):
    table._check(p)
    assert len(step_sizes) == len(lr_wds) == table.n_groups
    if clip_sumsq is not None:      # read once, before any segment is updated (as the kernel does)
        clip_sumsq = clip_sumsq.clone()
    for a, length, grp in table.host.tolist():
        sl = slice(a, a + length)
        fake_ops.adamw_step(p[sl], g[sl], m[sl], v[sl], None if p_bf16 is None else p_bf16[sl],
                            step_size=step_sizes[grp], beta1=beta1, beta2=beta2, eps=eps,
                            lr_wd=lr_wds[grp], grad_scale=grad_scale, clip_sumsq=clip_sumsq,
                            clip_max_norm=clip_max_norm)


def sumsq_segments(x, table, out):
    table._check(x)
    acc = x.new_zeros((), dtype=x.dtype).double()
    for a, length, _ in table.host.tolist():
        acc = acc + (x[a:a + length].double() ** 2).sum()
    out.add_(acc.float())
    return out


def install(monkeypatch):
    """fake_ops.install plus the segment-table entry points."""
    from hero_b200 import ops
    fake_ops.install(monkeypatch)
    for name in ("adamw_step_groups", "sumsq_segments"):
        monkeypatch.setattr(ops, name, globals()[name])
