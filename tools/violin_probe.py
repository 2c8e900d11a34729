"""VIOLIN measurements on one GPU: training step of HeroForViolin (fwd + bwd + FusedAdamW) on the
syn_violin preset against the reference's HeroForViolin (staged under oracle/_ref, bf16 autocast,
torch fused AdamW) with the two arms alternated, per-call times of the pooling kernels in
single-pooling mode and of the two-pooling call at Nq = 1, validate_violin throughput, and the
share of joint rows that take the long-row attention path. The card's name and power limit are
read in the same run and name the output file (tools/violin_probe_<card>_<watts>w.json).

    python tools/violin_probe.py [--out-dir tools]
"""
import argparse
import json
import os
import re
import sys

import torch
from torch.nn import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import evalpass, ops, synth  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.optim import FusedAdamW  # noqa: E402
from hero_b200.params import flat_of  # noqa: E402
from hero_b200.plan import QA_PLAN_KEY, attach_plan  # noqa: E402
from hero_b200.violin import HeroForViolin  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import stage_ref  # noqa: E402
from tools.videoqa_probe import card, config_path, events_ms  # noqa: E402

DEV = torch.device("cuda")


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"violin_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def ours_step(batches):
    torch.manual_seed(0)
    model = HeroForViolin(VideoModelConfig(config_path()), 4352, 100).to(DEV).train()
    flat = flat_of(model, DEV)
    flat.mark_dirty()
    opt = FusedAdamW(flat, lr=1e-5)

    def step(i):
        opt.zero_grad()
        model(batches[i % len(batches)], "violin").backward()
        opt.step()
    return model, step


def reference_step(batches):
    gg.REF = stage_ref.available()
    gg.install_stubs()
    from model.model import VideoModelConfig as RefConfig
    from model.violin import HeroForViolin as RefViolin
    torch.manual_seed(0)
    model = RefViolin(RefConfig(config_path()), vfeat_dim=4352, max_frm_seq_len=100).to(DEV)
    model.train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-5, fused=True)

    def step(i):
        b = batches[i % len(batches)]
        opt.zero_grad(set_to_none=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = model(dict(b), "violin", compute_loss=False)
        # the reference's loss expression, outside autocast: torch refuses binary_cross_entropy
        # under CUDA autocast
        F.binary_cross_entropy(torch.sigmoid(logits.float()).squeeze(-1),
                               b["targets"].squeeze(-1).float()).backward()
        opt.step()
    return step


def pool_times(rows, length, H):
    h = torch.randn(rows * length + 64, H, device=DEV)
    fmap = torch.arange(rows * length, dtype=torch.int32, device=DEV)
    mask = torch.ones(rows * length, device=DEV)
    w = torch.randn(H, device=DEV) * 0.02
    a, b = torch.empty(rows * length, device=DEV), torch.empty(rows * length, device=DEV)
    qa, sp = torch.empty(rows, H, device=DEV), torch.empty(rows * length, H, device=DEV)
    dh = torch.zeros_like(h)
    dw1, dw2 = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    calls = {
        "single_fwd": lambda i: ops.qa_pool_fwd(h, fmap, mask, w, None, rows, 1, length, a, None,
                                                qa, None),
        "single_bwd": lambda i: ops.qa_pool_bwd(h, fmap, mask, w, None, a, None, qa, None, rows,
                                                1, length, dh, dw1, None),
        "two_pool_fwd": lambda i: ops.qa_pool_fwd(h, fmap, mask, w, w, rows, 1, length, a, b, qa,
                                                  sp),
        "two_pool_bwd": lambda i: ops.qa_pool_bwd(h, fmap, mask, w, w, a, b, qa, sp, rows, 1,
                                                  length, dh, dw1, dw2),
    }
    for fn in calls.values():
        events_ms(fn, 20)
    return {k: events_ms(fn, 500) for k, fn in calls.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    args = ap.parse_args()
    name, watts = card()
    host = [attach_plan(synth.syn_violin(seed=s), kind="violin") for s in range(4)]
    ours_b = [synth.to_device(b, DEV) for b in host]
    long_rows = sum(b[QA_PLAN_KEY].n_long_rows for b in host)
    rows = sum(b[QA_PLAN_KEY].seq.rows for b in host)
    model, ours = ours_step(ours_b)
    arms = {"ours": ours}
    if stage_ref.available():
        ref_b = [synth.to_device({k: v for k, v in b.items() if not k.startswith("_hero")}, DEV)
                 for b in host]
        arms["reference_bf16_autocast"] = reference_step(ref_b)
    for fn in arms.values():
        events_ms(fn, args.warmup)
    times = {k: [] for k in arms}
    for _ in range(args.repeats):                      # alternate the arms
        for k, fn in arms.items():
            times[k].append(events_ms(fn, args.steps))
    # pooling per call at the preset's shape: 8 rows, L 100, H 768
    pool_ms = pool_times(8, 100, 768)
    # evaluation throughput: val_batch_size 10 (config/train-violin-8gpu.json), one statement each
    loader = []
    for s in range(8):
        vb = attach_plan(synth.syn_violin_batch(n_videos=10, n_statements=1, seed=100 + s),
                         kind="violin")
        vb = synth.to_device(vb, DEV)
        vb["qids"] = list(range(10 * s, 10 * s + 10))
        loader.append(vb)
    evalpass.validate_violin(model, [dict(loader[0])], "val")
    torch.cuda.synchronize()
    val_log, _, _ = evalpass.validate_violin(model, [dict(b) for b in loader], "val")
    out = {"gpu": name, "power_limit": watts,
           "preset": "syn_violin: 4 statement pairs = 8 rows, clips of 20-100 frames",
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
           "step_ms": times,
           "step_ms_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
           "pool_shape": "rows 8, Nq 1, L 100, H 768",
           "pool_ms_per_call": pool_ms,
           "validate_statements_per_s": val_log["valid/val_ex_per_s"],
           "validate_batch": "10 statements, 8 batches",
           "long_rows": long_rows, "joint_rows": rows, "long_row_share": long_rows / rows}
    print(json.dumps(out, indent=1))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
