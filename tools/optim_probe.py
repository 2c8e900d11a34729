"""FusedAdamW with the reference's four parameter groups on one GPU: time of `step()` on the flat
buffer of the real fine-tuning model (HeroForVideoQA, 6 + 3 layers, H 768, vocabulary 50 272) with
lr_mul = 10 (config/train-tvqa-8gpu.json), four arms alternated, CUDA events after warm-up:

  grouped     one hero_adamw_step_groups launch over the optimizer's segment table
  per_range   the same update as one hero_adamw_step launch per flat range of the four groups
  reference   the reference's optim/adamw.py AdamW with the four groups of its own
              optim/misc.py build_optimizer (staged under oracle/_ref), over the same parameters
  step_call   the whole FusedAdamW.step() call (its host work included: ensure_flat_grads
              re-checks every parameter's .grad view, which a training step overlaps with the
              device work of forward / backward)

It also checks that the grouped and per-range updates are bitwise equal at this size, and reads
the card's name, power limit and the SM / memory clocks it held while a timed window ran. The
output file is named after the card and power limit (tools/optim_probe_<card>_<watts>w.json).

    python tools/optim_probe.py [--steps 50] [--repeats 5] [--out-dir tools]
"""
import argparse
import json
import math
import os
import re
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import ops  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.optim import build_optimizer  # noqa: E402
from hero_b200.videoqa import HeroForVideoQA  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import stage_ref  # noqa: E402
from tools.videoqa_probe import card, config_path, events_ms  # noqa: E402

DEV = torch.device("cuda")
BYTES_PER_PARAM = 30     # p, g, m, v read; p, m, v and the bf16 mirror written


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"optim_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def clocks_under_load(fn, n):
    """SM / memory clocks read by nvidia-smi while n calls of fn are queued on the GPU."""
    for i in range(n):
        fn(i)
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.mem,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    torch.cuda.synchronize()
    sm, mem, max_sm = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"sm": sm, "mem": mem, "max_sm": max_sm}


def step_sizes(opt, t):
    """FusedAdamW.step()'s per-group (step_size, lr * weight_decay) at step t."""
    b1, b2 = opt.betas
    return [(grp["lr"] * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t),
             grp["lr"] * grp["weight_decay"]) for grp in opt.param_groups]


def grouped_step(opt):
    def step(_):
        opt.step_count += 1
        sizes = step_sizes(opt, opt.step_count)
        ops.adamw_step_groups(opt.flat.flat, opt.flat.grad_flat, opt.exp_avg, opt.exp_avg_sq,
                              opt.flat.mirror, opt._segments, step_sizes=[s for s, _ in sizes],
                              lr_wds=[w for _, w in sizes], beta1=opt.betas[0],
                              beta2=opt.betas[1], eps=opt.eps)
    return step


def per_range_step(opt):
    """The grouped update as one hero_adamw_step per flat range (same step sizes)."""
    def step(_):
        opt.step_count += 1
        g = opt.flat.grad_flat
        for grp, (step_size, lr_wd) in zip(opt.param_groups, step_sizes(opt, opt.step_count)):
            for a, b in grp["ranges"]:
                ops.adamw_step(opt.flat.flat[a:b], g[a:b], opt.exp_avg[a:b], opt.exp_avg_sq[a:b],
                               opt.flat.mirror[a:b], step_size=step_size, beta1=opt.betas[0],
                               beta2=opt.betas[1], eps=opt.eps, lr_wd=lr_wd)
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    args = ap.parse_args()
    name, watts = card()

    torch.manual_seed(0)
    model = HeroForVideoQA(VideoModelConfig(config_path()), 4352, 100).to(DEV).train()
    opts = types.SimpleNamespace(optim="adamw", learning_rate=5e-5, lr_mul=10.0,
                                 betas=[0.9, 0.98], weight_decay=0.01)
    opt = build_optimizer(model, opts)
    flat = opt.flat
    assert len(opt.param_groups) == 4
    g = torch.Generator(device=DEV).manual_seed(1)
    flat.grad_flat.copy_(torch.randn(flat.total, device=DEV, generator=g) * 1e-3)
    ranges = sum(len(grp["ranges"]) for grp in opt.param_groups)

    # bitwise: grouped launch == per-range launches, from the same state
    state = [t.clone() for t in (flat.flat, opt.exp_avg, opt.exp_avg_sq, flat.mirror)]
    opt.step()
    grouped = [t.clone() for t in (flat.flat, opt.exp_avg, opt.exp_avg_sq, flat.mirror)]
    for t, s in zip((flat.flat, opt.exp_avg, opt.exp_avg_sq, flat.mirror), state):
        t.copy_(s)
    opt.step_count = 0
    per_range_step(opt)(0)
    bitwise = all(torch.equal(a, b) for a, b in
                  zip(grouped, (flat.flat, opt.exp_avg, opt.exp_avg_sq, flat.mirror)))
    del state, grouped

    arms = {"grouped": grouped_step(opt), "per_range": per_range_step(opt),
            "step_call": lambda i: opt.step()}
    if stage_ref.available():
        gg.REF = stage_ref.available()
        gg.install_stubs()
        from optim.misc import build_optimizer as ref_build_optimizer
        ref_opt = ref_build_optimizer(model, opts)      # the same parameters and gradients
        arms["reference"] = lambda i: ref_opt.step()
    for fn in arms.values():
        events_ms(fn, args.warmup)
    times = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            times[k].append(events_ms(fn, args.steps))
    clocks = clocks_under_load(arms["grouped"], 1000)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    covered = opt._segments.covered
    out = {"gpu": name, "power_limit": watts, "clocks_during_grouped_steps": clocks,
           "model": "HeroForVideoQA, 6 + 3 layers, H 768, vocabulary 50272; lr_mul 10",
           "flat_total": flat.total, "params_in_groups": covered,
           "groups": [{"lr": grp["lr"], "weight_decay": grp["weight_decay"],
                       "ranges": len(grp["ranges"]),
                       "elements": sum(b - a for a, b in grp["ranges"])}
                      for grp in opt.param_groups],
           "per_range_launches": ranges,
           "grouped_bitwise_equal_to_per_range": bitwise,
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
           "step_ms": times, "step_ms_median": med,
           "grouped_hbm_gb_per_s": BYTES_PER_PARAM * covered / (med["grouped"] * 1e-3) / 1e9}
    print(json.dumps(out, indent=1))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
