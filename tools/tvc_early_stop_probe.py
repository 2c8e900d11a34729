"""TVC early stop on one GPU: ms per batch of TvcGenerator greedy decoding, beam search B = 5 and
sample(top_p=0.9), each with early_stop off and on, on syn_tvc_val (8 videos, 2-6 caption segments
each) at real dimensions (6 + 3 encoder layers, 2 decoder layers, H 768, vocabulary 50 272), in two
kinds of case:

  no_end        EOS biased by -1000 so that no row ever ends, max_step 30: what the extra launch
                per step costs when nothing stops (the worst case)
  m<m>_T<T>     every row ends at step m (min_length = m and EOS biased by +1000), m in {10, 20},
                max_step 30 and 60

A randomly initialised decoder almost never emits EOS, hence the bias. Within a case every shape is
warmed up and the arms are alternated, their order rotated by one arm per repeat; the medians of the
repeats are reported. For every early-stopped arm, a separate untimed pass counts the steps the host
enqueued after the device's stop step (it stops on the first poll that sees the step, so the count
is how far ahead of the device it was). The card's name and power limit are read in the same run
and name the output file (tools/tvc_early_stop_probe_<card>_<watts>w.json).

    python tools/tvc_early_stop_probe.py [--out-dir tools]
"""
import argparse
import json
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import ops, synth  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.plan import attach_plan  # noqa: E402
from hero_b200.tvc import HeroForTvc, TvcGenerator  # noqa: E402
from tools.tvc_probe import config_path  # noqa: E402
from tools.videoqa_probe import card, events_ms  # noqa: E402

DEV = torch.device("cuda")
BIAS = 1000.0
CASES = {"no_end": (-BIAS, 0, 30), "m10_T30": (BIAS, 10, 30), "m20_T30": (BIAS, 20, 30),
         "m10_T60": (BIAS, 10, 60), "m20_T60": (BIAS, 20, 60)}


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"tvc_early_stop_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def strategies(gen, pick):
    return {"greedy": lambda i: gen.greedy_decode(pick(i)),
            "beam5": lambda i: gen.beam_search(pick(i), 5),
            "sample_top_p0.9": lambda i: gen.sample(pick(i), top_p=0.9, seed=i)}


def steps_beyond_stop(fn, n):
    """Per call of fn(0 .. n - 1): the steps the host enqueued after the device's stop step (None
    without a stop)."""
    inner, out = ops.dec_finished, []
    seen = {}

    def spy(ids, fin, stop_dev, stop_host, **kw):
        seen["n"] = kw["step"] + 1
        seen["dev"] = stop_dev
        inner(ids, fin, stop_dev, stop_host, **kw)
    ops.dec_finished = spy
    try:
        for i in range(n):
            fn(i)
            stop = int(seen["dev"])
            out.append(None if stop == ops.DEC_STOP_UNSET else seen["n"] - 1 - stop)
    finally:
        ops.dec_finished = inner
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    args = ap.parse_args()
    name, watts = card()
    torch.manual_seed(0)
    model = HeroForTvc(VideoModelConfig(config_path()), 4352, 100).to(DEV).eval()
    host = [attach_plan(synth.syn_tvc_val(seed=s)) for s in range(args.batches)]
    n_caps = [len(b["clip_ids"]) for b in host]
    dev_b = [synth.to_device(b, DEV) for b in host]
    pick = lambda i: dev_b[i % len(dev_b)]   # noqa: E731
    bias = model.v_encoder.f_encoder.lm_head.bias
    eos_base = float(bias.detach()[synth.EOS])
    res = {}
    for case, (b, m, T) in CASES.items():
        with torch.no_grad():
            bias[synth.EOS] = eos_base + b
        arms = {}
        for stop in (False, True):
            gen = TvcGenerator(model, T, synth.BOS, synth.EOS, fp16=False, min_length=m,
                               early_stop=stop)
            for k, fn in strategies(gen, pick).items():
                arms[f"{k}/{'on' if stop else 'off'}"] = fn
        for fn in arms.values():                        # every batch shape, every arm
            for i in range(max(args.warmup, 1) * len(dev_b)):
                fn(i)
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        names = list(arms)
        for r in range(args.repeats):                   # alternate the arms, rotating the order
            for k in names[r % len(names):] + names[:r % len(names)]:
                times[k].append(events_ms(arms[k], args.batches))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        res[case] = {
            "eos_bias": b, "min_length": m, "max_step": T, "ms_per_batch": times,
            "ms_per_batch_median": med,
            "on_over_off": {k.split("/")[0]: med[k] / med[k.replace("/on", "/off")]
                            for k in med if k.endswith("/on")},
            "steps_enqueued_beyond_stop": {k.split("/")[0]: steps_beyond_stop(arms[k],
                                                                              args.batches)
                                           for k in arms if k.endswith("/on")}}
        print(case, json.dumps({k: round(v, 3) for k, v in med.items()}), flush=True)
    out = {"gpu": name, "power_limit": watts,
           "preset": "syn_tvc_val: 8 videos of 20-100 frames, 2-6 caption segments each "
                     "(one empty); 6 + 3 encoder layers, 2 decoder layers, H 768, vocabulary "
                     "50272, randomly initialised (EOS forced or suppressed by its LM-head bias)",
           "captions_per_batch": n_caps, "batches": args.batches, "warmup": args.warmup,
           "repeats": args.repeats,
           "order": "within a case, repeat r starts at arm r mod 6 of the case's arms",
           "cases": res}
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({c: v["on_over_off"] for c, v in res.items()}, indent=1))


if __name__ == "__main__":
    main()
