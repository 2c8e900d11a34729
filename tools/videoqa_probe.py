"""Video QA measurements on one GPU: training step of HeroForVideoQA (fwd + bwd + fused AdamW) on
the TVQA preset against the reference's HeroForVideoQA (staged under oracle/_ref, bf16 autocast,
torch fused AdamW) with the two arms alternated, per-launch times of the pooling kernels,
validate_videoqa throughput, and the share of joint rows that take the long-row attention path.
The card's name and power limit are read in the same run.

    python tools/videoqa_probe.py --out tools/videoqa_probe_h100_400w.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import evalpass, synth  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.optim import FusedAdamW  # noqa: E402
from hero_b200.params import flat_of  # noqa: E402
from hero_b200.plan import QA_PLAN_KEY, attach_plan  # noqa: E402
from hero_b200.videoqa import HeroForVideoQA  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import stage_ref  # noqa: E402

DEV = torch.device("cuda")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, watts = [s.strip() for s in q.split(",")]
    return name, watts


def events_ms(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(n):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def config_path():
    f = tempfile.NamedTemporaryFile("w", suffix=".json", delete=False)
    json.dump(gg.model_json(768, 3072, 12, 6, 3, 50272), f)
    f.close()
    return f.name


def ours_step(batches):
    torch.manual_seed(0)
    model = HeroForVideoQA(VideoModelConfig(config_path()), 4352, 100).to(DEV).train()
    flat = flat_of(model, DEV)
    flat.mark_dirty()
    opt = FusedAdamW(flat, lr=1e-5)

    def step(i):
        opt.zero_grad()
        qa, t = model(batches[i % len(batches)], "tvqa")
        (qa + 0.4 * t).backward()
        opt.step()
    return model, step


def reference_step(batches):
    gg.REF = stage_ref.available()
    gg.install_stubs()
    from model.model import VideoModelConfig as RefConfig
    from model.videoQA import HeroForVideoQA as RefQA
    torch.manual_seed(0)
    model = RefQA(RefConfig(config_path()), vfeat_dim=4352, max_frm_seq_len=100).to(DEV).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-5, fused=True)

    def step(i):
        opt.zero_grad(set_to_none=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            qa, t = model(dict(batches[i % len(batches)]), "tvqa")
        (qa + 0.4 * t).backward()
        opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "videoqa_probe_h100.json"))
    args = ap.parse_args()
    name, watts = card()
    host = [attach_plan(synth.syn_tvqa(seed=s), kind="videoqa") for s in range(4)]
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
    # pooling kernels per launch, TVQA shapes (Nv 4, Nq 5, L 100, H 768)
    from hero_b200 import ops
    nv, nq, length, H = 4, 5, 100, 768
    h = torch.randn(nv * nq * length + 64, H, device=DEV)
    fmap = torch.arange(nv * nq * length, dtype=torch.int32, device=DEV)
    mask = torch.ones(nv * nq * length, device=DEV)
    w = torch.randn(H, device=DEV) * 0.02
    a, b = torch.empty(nv * nq * length, device=DEV), torch.empty(nv * nq * length, device=DEV)
    qa, sp = torch.empty(nv * nq, H, device=DEV), torch.empty(nv * length, H, device=DEV)
    dh = torch.zeros_like(h)
    dw1, dw2 = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    fwd = lambda i: ops.qa_pool_fwd(h, fmap, mask, w, w, nv, nq, length, a, b, qa, sp)
    bwd = lambda i: ops.qa_pool_bwd(h, fmap, mask, w, w, a, b, qa, sp, nv, nq, length, dh, dw1, dw2)
    events_ms(fwd, 20)
    events_ms(bwd, 20)
    pool_fwd_ms, pool_bwd_ms = events_ms(fwd, 200), events_ms(bwd, 200)
    # evaluation throughput
    loader = []
    for s in range(8):
        vb = attach_plan(synth.syn_videoqa_batch(n_videos=10, n_cand=5, seed=100 + s),
                         kind="videoqa")
        vb = synth.to_device(vb, DEV)
        vb["qids"] = list(range(10 * s, 10 * s + 10))
        loader.append(vb)
    evalpass.validate_videoqa(model, [dict(loader[0])], "val")
    torch.cuda.synchronize()
    val_log, _, _ = evalpass.validate_videoqa(model, [dict(b) for b in loader], "val")
    out = {"gpu": name, "power_limit": watts, "preset": "syn_tvqa: 4 videos x 5 candidates",
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
           "step_ms": times,
           "step_ms_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
           "qa_pool_fwd_ms": pool_fwd_ms, "qa_pool_bwd_ms": pool_bwd_ms,
           "validate_questions_per_s": val_log["valid/ex_per_s"],
           "validate_batch": "10 videos x 5 candidates, 8 batches",
           "long_rows": long_rows, "joint_rows": rows, "long_row_share": long_rows / rows}
    print(json.dumps(out, indent=1))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
