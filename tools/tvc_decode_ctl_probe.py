"""TVC decoding controls on one GPU: ms per batch of TvcGenerator greedy decoding, greedy with
no_repeat_ngram_size 3 and min_length 5, beam search B = 5 without and with the same controls, and
sample(top_p=0.9), on syn_tvc_val (8 videos, 2-6 caption segments each, max_step 30) at real
dimensions (6 + 3 encoder layers, 2 decoder layers, H 768, vocabulary 50 272), every shape warmed
up and the arms alternated, their order rotated by one arm per repeat so that no arm always runs
first; and the device time per launch of hero_dec_ban_tokens and
hero_sample_tokens against rank_topk(k=1) on the same logits rows, from torch.profiler in a child
process with HERO_SERIAL_PROFILE=1 (with programmatic dependent launch a kernel's recorded duration
would include its wait on the one before it). The card's name and power limit are read in the same
run and name the output file (tools/tvc_decode_ctl_probe_<card>_<watts>w.json).

    python tools/tvc_decode_ctl_probe.py [--out-dir tools]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import ops, synth  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.plan import attach_plan  # noqa: E402
from hero_b200.tvc import HeroForTvc, TvcGenerator  # noqa: E402
from tools.tvc_beam_probe import device_us  # noqa: E402
from tools.tvc_probe import config_path  # noqa: E402
from tools.videoqa_probe import card, events_ms  # noqa: E402

DEV = torch.device("cuda")
MAX_STEP = 30
CONTROLS = dict(no_repeat_ngram_size=3, min_length=5)


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"tvc_decode_ctl_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def kernel_device_us(rows, n_valid, ld):
    """Device time per launch (us) of the three per-step selections on the same rows: rank_topk
    (k = 1), ban_tokens (n = 3, min_length 5, at a late step of a 30-step history, and at the
    longest history, 1023 steps) and sample_tokens (top_p 0.9; top_k 50 + top_p 0.9)."""
    gen = torch.Generator().manual_seed(0)
    logits = (3 * torch.randn(rows, ld, generator=gen)).to(DEV)
    vals = torch.empty(rows, 1, device=DEV)
    idx = torch.empty(rows, 1, dtype=torch.int32, device=DEV)
    ids = torch.empty(rows, dtype=torch.int32, device=DEV)
    out = {"rows": rows, "columns": n_valid,
           "rank_topk_k1": device_us(lambda i: ops.rank_topk(logits, n_valid, 1, vals, idx),
                                     "rank_topk")}
    for T, step in ((MAX_STEP, MAX_STEP - 1), (1023, 1022)):
        hist = torch.randint(3, 40, (T, rows), generator=gen).int().to(DEV)
        out[f"ban_tokens_step{step}"] = device_us(
            lambda i: ops.ban_tokens(logits, n_valid, hist, step_stride=rows, row_stride=1, bos=0,
                                     step=step, ngram=3, min_length=5, eos=2), "ban_tokens")
    for name, kw in (("sample_tokens_top_p0.9", dict(top_k=0, top_p=0.9)),
                     ("sample_tokens_top_k50_top_p0.9", dict(top_k=50, top_p=0.9)),
                     ("sample_tokens_plain", dict(top_k=0, top_p=1.0))):
        out[name] = device_us(lambda i: ops.sample_tokens(logits, n_valid, ids, temperature=1.0,
                                                          seed=1, step=i, **kw), "sample_tokens")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    ap.add_argument("--device-times", type=int, default=0,
                    help="(child process) print the kernels' device times at this row count")
    ap.add_argument("--n-valid", type=int, default=50265)
    ap.add_argument("--ld", type=int, default=50272)
    args = ap.parse_args()
    if args.device_times:
        res = {"greedy_rows": kernel_device_us(args.device_times, args.n_valid, args.ld),
               "beam5_rows": kernel_device_us(5 * args.device_times, args.n_valid, args.ld)}
        print(json.dumps(res))
        return
    name, watts = card()
    torch.manual_seed(0)
    model = HeroForTvc(VideoModelConfig(config_path()), 4352, 100).to(DEV).eval()
    host = [attach_plan(synth.syn_tvc_val(seed=s)) for s in range(args.batches)]
    n_caps = [len(b["clip_ids"]) for b in host]
    dev_b = [synth.to_device(b, DEV) for b in host]
    plain = TvcGenerator(model, MAX_STEP, synth.BOS, synth.EOS, fp16=False)
    ctl = TvcGenerator(model, MAX_STEP, synth.BOS, synth.EOS, fp16=False, **CONTROLS)
    pick = lambda i: dev_b[i % len(dev_b)]   # noqa: E731
    arms = {
        "greedy": lambda i: plain.greedy_decode(pick(i)),
        "greedy_ngram3_min5": lambda i: ctl.greedy_decode(pick(i)),
        "beam5": lambda i: plain.beam_search(pick(i), 5),
        "beam5_ngram3_min5": lambda i: ctl.beam_search(pick(i), 5),
        "sample_top_p0.9": lambda i: plain.sample(pick(i), top_p=0.9, seed=i),
    }
    for fn in arms.values():                            # every batch shape, every arm
        for i in range(max(args.warmup, 1) * len(dev_b)):
            fn(i)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    names = list(arms)
    for r in range(args.repeats):                       # alternate the arms, rotating the order
        for k in names[r % len(names):] + names[:r % len(names)]:
            times[k].append(events_ms(arms[k], args.batches))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    fe = model.v_encoder.f_encoder
    n_valid = fe.embeddings.word_embeddings.weight.shape[0] - fe.vocab_pad
    env = dict(os.environ, HERO_SERIAL_PROFILE="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--device-times",
                        str(max(n_caps)), "--n-valid", str(n_valid),
                        "--ld", str(fe.embeddings.word_embeddings.weight.shape[0])],
                       env=env, capture_output=True, text=True, check=True)
    serial = json.loads(r.stdout.strip().splitlines()[-1])
    out = {"gpu": name, "power_limit": watts,
           "preset": "syn_tvc_val: 8 videos of 20-100 frames, 2-6 caption segments each "
                     "(one empty), max_step 30; 6 + 3 encoder layers, 2 decoder layers, H 768, "
                     "vocabulary 50272",
           "controls": CONTROLS, "captions_per_batch": n_caps, "batches": args.batches,
           "warmup": args.warmup, "repeats": args.repeats,
           "order": "repeat r starts at arm r mod 5 of " + ", ".join(names),
           "ms_per_batch": times,
           "ms_per_batch_median": med, "kernel_device_us": serial}
    print(json.dumps(out, indent=1))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
