"""Fused AdamW over the flat parameter buffer, with the reference's exact update rule
(optim/adamw.py:80-104) and parameter grouping (optim/misc.py:14-50): eps 1e-6 added to
sqrt(v), bias-corrected step size, decoupled weight decay applied after the Adam update with
the un-corrected lr, no decay for names containing 'bias' / 'LayerNorm.*'.

The reference launches ~10 pointwise kernels for each of ~208 tensors per step; here the flat
layout (decayed parameters first, see params.py) needs TWO launches, and the same kernel refreshes
the bf16 working copy so the next forward skips its cast pass.

With the reference's four groups (`lr_mul` != 1 or frozen parameters, see `build_optimizer`),
each group is a list of flat ranges, and a step is ONE launch over a segment table uploaded when
the optimizer is built; the groups' step sizes travel as kernel arguments, so changing a group's
`lr` between steps costs no copy and no synchronisation.
"""
import math

import torch

from . import ops
from .params import FlatParams, is_no_decay


class FusedAdamW:
    """`groups=None`: two flat ranges over the whole buffer (decay / no-decay) with one learning
    rate, two launches per step. Otherwise `groups` is a list of at most ops.ADAMW_MAX_GROUPS
    {"lr", "weight_decay", "ranges": [(start, end), ...]}, ranges disjoint with multiple-of-4
    bounds: one launch per step, and elements in no range are never updated and not counted by
    gradient clipping."""

    def __init__(self, flat, lr=1e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01,
                 correct_bias=True, groups=None):
        assert isinstance(flat, FlatParams) and flat.flat is not None, \
            "call flat_of(model, device) (or run one forward) before building the optimizer"
        self.flat = flat
        self._generation = flat.generation
        self.correct_bias = correct_bias
        self.eps = eps
        self.betas = betas
        # `param_groups` keeps the reference loops working:
        #     for g in optimizer.param_groups: g['lr'] = lr_this_step   (train_vcmr.py:245-247)
        #     groups 0 / 1 at lr * lr_mul, 2 / 3 at lr                   (train_videoQA.py:186-192)
        if groups is None:
            split = flat.no_decay_start
            self.param_groups = [
                {"lr": lr, "weight_decay": weight_decay, "range": (0, split)},
                {"lr": lr, "weight_decay": 0.0, "range": (split, flat.total)},
            ]
            self._segments = None
        else:
            self.param_groups = [{"lr": float(g["lr"]), "weight_decay": float(g["weight_decay"]),
                                  "ranges": [(int(a), int(b)) for a, b in g["ranges"]]}
                                 for g in groups]
            self._segments = ops.SegmentTable(
                [(a, b - a, i) for i, g in enumerate(self.param_groups) for a, b in g["ranges"]],
                flat.total, len(self.param_groups), flat.flat.device)
        # some element of the buffer belongs to no group: clip over the segments only
        self._partial = self._segments is not None and self._segments.covered < flat.total
        self.exp_avg = torch.zeros_like(flat.flat)
        self.exp_avg_sq = torch.zeros_like(flat.flat)
        self.step_count = 0
        flat.ensure_flat_grads()

    def zero_grad(self, set_to_none=False):
        self.flat.ensure_flat_grads().zero_()

    def _add_sumsq(self, g, out):
        if self._partial:
            ops.sumsq_segments(g, self._segments, out)
        else:
            ops.sumsq(g, out)

    def grad_norm(self):
        g = self.flat.ensure_flat_grads()
        acc = torch.zeros(1, dtype=torch.float32, device=g.device)
        self._add_sumsq(g, acc)
        return acc.sqrt()

    def clip_grad_norm_(self, max_norm):
        """Global-norm clip folded into the update (train_vcmr.py:258-259): returns the norm and
        remembers the scale for the next step()."""
        total = float(self.grad_norm().item())
        self._grad_scale = min(1.0, max_norm / (total + 1e-6))
        return total

    def clip_grad_norm_device_(self, max_norm):
        """Global-norm clip (train_vcmr.py:258-259) with no device->host read: the sum of squares
        stays on the device and the next step()'s AdamW kernels scale the gradients by
        min(1, max_norm / (norm + 1e-6)) themselves. Returns the device scalar (sum of squares)."""
        g = self.flat.ensure_flat_grads()
        if getattr(self, "_sumsq", None) is None:
            self._sumsq = torch.zeros(1, dtype=torch.float32, device=g.device)
        self._sumsq.zero_()
        self._add_sumsq(g, self._sumsq)
        self._clip = float(max_norm)
        return self._sumsq

    def step(self):
        if self.flat.generation != self._generation or self.exp_avg.numel() != self.flat.total:
            raise RuntimeError("the parameters were re-flattened (a module was replaced or moved) "
                               "after this optimizer was built: its moment buffers and ranges no "
                               "longer describe the flat buffer; rebuild the optimizer")
        self.step_count += 1
        t = self.step_count
        b1, b2 = self.betas
        g = self.flat.ensure_flat_grads()
        scale = getattr(self, "_grad_scale", 1.0)
        self._grad_scale = 1.0
        clip = getattr(self, "_clip", None)
        self._clip = None
        clip_args = dict(grad_scale=scale, clip_sumsq=self._sumsq if clip is not None else None,
                         clip_max_norm=clip or 0.0)
        if self._segments is not None:
            step_sizes, lr_wds = [], []
            for grp in self.param_groups:
                lr = grp["lr"]
                step_size = lr
                if self.correct_bias:
                    step_size = lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
                step_sizes.append(step_size)
                lr_wds.append(lr * grp["weight_decay"])
            ops.adamw_step_groups(self.flat.flat, g, self.exp_avg, self.exp_avg_sq,
                                  self.flat.mirror, self._segments, step_sizes=step_sizes,
                                  lr_wds=lr_wds, beta1=b1, beta2=b2, eps=self.eps, **clip_args)
        else:
            for grp in self.param_groups:
                a, b = grp["range"]
                if b <= a:
                    continue
                lr = grp["lr"]
                step_size = lr
                if self.correct_bias:
                    step_size = lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
                ops.adamw_step(self.flat.flat[a:b], g[a:b], self.exp_avg[a:b],
                               self.exp_avg_sq[a:b], self.flat.mirror[a:b], step_size=step_size,
                               beta1=b1, beta2=b2, eps=self.eps, lr_wd=lr * grp["weight_decay"],
                               **clip_args)
        # masters changed in place through a flat view: the mirror is already fresh
        self.flat.dirty = False
        self.flat._version_sum = sum(p._version for _, p, _, _ in self.flat._probe)

    def state_dict(self):
        return {"step": self.step_count, "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq,
                "param_groups": [{k: v for k, v in g.items()} for g in self.param_groups]}

    def load_state_dict(self, sd):
        if len(sd["param_groups"]) != len(self.param_groups):
            raise ValueError(f"optimizer state has {len(sd['param_groups'])} parameter groups, "
                             f"this optimizer has {len(self.param_groups)}")
        self.step_count = sd["step"]
        self.exp_avg.copy_(sd["exp_avg"])
        self.exp_avg_sq.copy_(sd["exp_avg_sq"])
        for g, s in zip(self.param_groups, sd["param_groups"]):
            g["lr"], g["weight_decay"] = s["lr"], s["weight_decay"]


def reference_groups(model, flat, opts):
    """The four groups of optim/misc.py:14-50 as flat ranges, in the reference's order: top (name
    without 'v_encoder') decay / no-decay at lr_mul * learning_rate, then v_encoder decay /
    no-decay at learning_rate. Names are those of `model.named_parameters()` (a tied weight counts
    once, under its first name), only parameters with `requires_grad` are members, and each member
    brings its alignment padding, so every range is a maximal run of whole parameters. Empty groups
    stay in the list: the training loops index them."""
    lr = float(opts.learning_rate)
    top_lr = float(getattr(opts, "lr_mul", 1.0)) * lr
    wd = float(opts.weight_decay)
    groups = [{"lr": top_lr, "weight_decay": wd, "ranges": []},
              {"lr": top_lr, "weight_decay": 0.0, "ranges": []},
              {"lr": lr, "weight_decay": wd, "ranges": []},
              {"lr": lr, "weight_decay": 0.0, "ranges": []}]
    named = {id(p): (n, p) for n, p in model.named_parameters()}
    ends = [off for _, _, off, _ in flat.entries[1:]] + [flat.total]   # entries are offset-ordered
    for (_, p, off, _), end in zip(flat.entries, ends):
        item = named.get(id(p))
        if item is None or not item[1].requires_grad:
            continue
        name = item[0]
        ranges = groups[(2 if "v_encoder" in name else 0) + (1 if is_no_decay(name) else 0)]["ranges"]
        if ranges and ranges[-1][1] == off:
            ranges[-1] = (ranges[-1][0], end)
        else:
            ranges.append((off, end))
    return groups


def build_optimizer(model, opts, device=None):
    """optim/misc.py:14-50 for optim == 'adamw' on the flat layout. With lr_mul == 1 and every
    parameter trainable, the reference's four groups share one learning rate and the update is
    that of the two flat ranges (decay / no-decay): a two-group FusedAdamW, two launches per step.
    Otherwise the result has the reference's four `param_groups` (`reference_groups`), which the
    fine-tuning loops index (`if i in (0, 1): lr *= lr_mul`, train_videoQA.py:186-192), and one
    launch per step.

    Frozen parameters (requires_grad False) belong to no group: they are never updated, their
    moments stay zero, their bf16 mirror entries are left as they are, and gradient clipping does
    not count them. The CUDA Functions still write their gradients into the flat gradient buffer,
    which is harmless but costs the work of computing them."""
    from .params import flat_of
    if getattr(opts, "optim", "adamw") != "adamw":
        raise ValueError(f"hero_b200.build_optimizer implements 'adamw' only (got {opts.optim!r}); "
                         "use the reference's torch optimizer for adam / adamax")
    device = device or next(model.parameters()).device
    flat = flat_of(model, device)
    grouped = float(getattr(opts, "lr_mul", 1.0)) != 1.0 or \
        any(not p.requires_grad for p in model.parameters())
    return FusedAdamW(flat, lr=opts.learning_rate, betas=tuple(opts.betas),
                      weight_decay=opts.weight_decay,
                      groups=reference_groups(model, flat, opts) if grouped else None)
