"""TVC caption metrics on one GPU against the reference's COCO scorers on the same host's CPU.

A synthetic validation split of 10 895 clips (1-4 references of 8-20 words, 6-16-word hypotheses,
Zipf vocabulary of 5 000 words; synth.syn_captions) is scored three ways in one run:

* the device pass of capeval (upload and kernels), by CUDA events over repeated calls after
  warm-up, and its kernels alone by torch.profiler;
* capeval.TVCEval(...)(records) end to end by the host clock, with ptb_tokenize's share measured
  separately (TVCEval tokenizes the references once, in its constructor; each call tokenizes the
  hypotheses);
* the reference's Bleu(4) / Rouge / Cider (eval/pycocoevalcap, staged by build() through
  oracle/stage_caption_scorers.py) on the same tokens.

The scores of both arms are compared. The card's name and power limit are read in the same run
and name the output file (tools/caption_metrics_probe_<card>_<watts>w.json).

    python tools/caption_metrics_probe.py [--out-dir tools]
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import capeval, synth  # noqa: E402
from tools.videoqa_probe import card, events_ms  # noqa: E402

N_CLIPS = 10895


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"caption_metrics_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def reference_arm(hyps, refs):
    from oracle import stage_caption_scorers
    root = stage_caption_scorers.available()
    if root is None:
        raise SystemExit("the reference's COCO scorers are not staged: run build() with a "
                         "readable reference checkout (oracle/stage_caption_scorers.py)")
    sys.path.insert(0, root)
    from pycocoevalcap.bleu.bleu import Bleu
    from pycocoevalcap.cider.cider import Cider
    from pycocoevalcap.rouge.rouge import Rouge
    gts = {i: [" ".join(r) for r in rs] for i, rs in enumerate(refs)}
    res = {i: [" ".join(h)] for i, h in enumerate(hyps)}
    out, secs = {}, {}
    for name, scorer in (("bleu", Bleu(4)), ("rouge", Rouge()), ("cider", Cider())):
        t = time.perf_counter()
        out[name] = scorer.compute_score(gts, res)[0]
        secs[name] = round(time.perf_counter() - t, 3)
    scores = dict(zip(capeval.METRICS, list(out["bleu"]) + [out["rouge"], out["cider"]]))
    return scores, secs


def kernel_ms(pack, reps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            capeval.device_stats(pack)
        torch.cuda.synchronize()
    ms = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count >= reps:
            ms[e.key[:60]] = round(e.device_time_total / 1e3 / reps, 4)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default="tools")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    name, watts = card()
    hyps, refs = synth.syn_captions(N_CLIPS, seed=0)

    # device pass
    pack = capeval.CaptionPack(hyps, refs)
    for _ in range(3):
        capeval.device_stats(pack)
    torch.cuda.synchronize()
    device_ms = events_ms(lambda i: capeval.device_stats(pack), args.reps)
    kernels = kernel_ms(pack, args.reps)
    t = time.perf_counter()
    for _ in range(args.reps):
        pack = capeval.CaptionPack(hyps, refs)
    pack_ms = (time.perf_counter() - t) / args.reps * 1e3
    t = time.perf_counter()
    for _ in range(args.reps):
        scores, _ = capeval.caption_scores(hyps, refs)
    caption_scores_ms = (time.perf_counter() - t) / args.reps * 1e3

    # TVCEval end to end, on caption text
    with tempfile.TemporaryDirectory() as td:
        ann = os.path.join(td, "ann.jsonl")
        with open(ann, "w") as f:
            for c, rs in enumerate(refs):
                f.write(json.dumps({"clip_id": c, "descs": [{"desc": " ".join(r).capitalize()
                                                             + "."} for r in rs]}) + "\n")
        records = [{"clip_id": c, "descs": [{"desc": " ".join(h).capitalize() + "."}]}
                   for c, h in enumerate(hyps)]
        t = time.perf_counter()
        ev = capeval.TVCEval(ann)
        ctor_s = time.perf_counter() - t
        ev(records)
        t = time.perf_counter()
        for _ in range(3):
            tvceval = ev(records)
        call_s = (time.perf_counter() - t) / 3
    t = time.perf_counter()
    for r in records:
        capeval.ptb_tokenize(r["descs"][0]["desc"])
    tok_hyp_s = time.perf_counter() - t

    ref_scores, ref_secs = reference_arm(hyps, refs)
    diff = {k: float(abs(scores[k] - ref_scores[k]) / max(abs(ref_scores[k]), 1e-300))
            for k in capeval.METRICS}
    out = {
        "card": name, "power_limit": watts, "clips": N_CLIPS,
        "references": int(sum(map(len, refs))),
        "words": int(pack.lens.sum()), "vocab": pack.vocab_size,
        "device_pass_ms": round(device_ms, 3),
        "kernels_ms_per_pass": kernels,
        "host_pack_ms": round(pack_ms, 2),
        "caption_scores_ms": round(caption_scores_ms, 2),
        "tvceval_constructor_s": round(ctor_s, 3),
        "tvceval_call_s": round(call_s, 3),
        "of_which_ptb_tokenize_hyps_s": round(tok_hyp_s, 3),
        "reference_cpu_s": ref_secs,
        "reference_cpu_total_s": round(sum(ref_secs.values()), 3),
        "scores": scores, "tvceval_x100": tvceval, "reference_scores": ref_scores,
        "relative_difference": diff,
        "bleu_rouge_identical": all(scores[k] == ref_scores[k] for k in capeval.METRICS[:5]),
    }
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
