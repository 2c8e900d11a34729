"""TVC greedy decoding on one GPU: ms per batch of TvcGenerator.greedy_decode on syn_tvc_val
(8 videos, 2-6 caption segments each, max_gen_step 30 of train-tvc-8gpu.json) at real dimensions
(6 + 3 encoder layers, 2 decoder layers, H 768, vocabulary 50 272), against the reference's
TvcGenerator (staged under oracle/_ref) under bf16 autocast, the two arms alternated; the
decoder-attention kernel's time per call at the decode-step and cross-attention shapes; and the
share of a decode step spent on the vocabulary GEMM + rank_topk argmax. The card's name and power
limit are read in the same run and name the output file (tools/tvc_probe_<card>_<watts>w.json).

    python tools/tvc_probe.py [--out-dir tools]
"""
import argparse
import json
import os
import re
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import ops, synth  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.plan import attach_plan  # noqa: E402
from hero_b200.tvc import HeroForTvc, TvcGenerator  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import stage_ref  # noqa: E402
from tools.videoqa_probe import card, events_ms  # noqa: E402

DEV = torch.device("cuda")
MAX_STEP = 30


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"tvc_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def config_path():
    j = gg.model_json(768, 3072, 12, 6, 3, 50272)
    j["d_config"] = dict(j["f_config"], num_hidden_layers=2, max_position_embeddings=1024,
                         type_vocab_size=1)
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(j, f)
        path = f.name
    return path


def reference_generator(state_dict):
    gg.REF = stage_ref.available()
    gg.install_stubs()
    from model.model import VideoModelConfig as RefConfig
    from model.tvc import HeroForTvc as RefTvc
    from model.tvc import TvcGenerator as RefGenerator
    ref = RefTvc(RefConfig(config_path()), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(state_dict)
    ref = ref.to(DEV).eval()
    gen = RefGenerator(ref, MAX_STEP, synth.BOS, synth.EOS, fp16=False)

    def run(b):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return gen.greedy_decode(dict(b))
    return run


def attn_ms(rows, heads, lens, off_stride):
    H = heads * 64
    n_kv = rows * off_stride + 1024
    qkv = torch.randn(n_kv, 3 * H, device=DEV).to(torch.bfloat16)
    off = (torch.arange(rows, device=DEV) * off_stride).int()
    ln = torch.full((rows,), lens, dtype=torch.int32, device=DEV)
    out = torch.empty(rows, H, dtype=torch.bfloat16, device=DEV)
    fn = lambda i: ops.dec_attn_fwd(qkv[:rows, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], off, ln,  # noqa
                                    out, heads=heads, max_kv_len=lens)
    events_ms(fn, 20)
    return events_ms(fn, 1000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    args = ap.parse_args()
    name, watts = card()
    torch.manual_seed(0)
    model = HeroForTvc(VideoModelConfig(config_path()), 4352, 100).to(DEV).eval()
    host = [attach_plan(synth.syn_tvc_val(seed=s)) for s in range(args.batches)]
    n_caps = [len(b["clip_ids"]) for b in host]
    ours_b = [synth.to_device(b, DEV) for b in host]
    gen = TvcGenerator(model, MAX_STEP, synth.BOS, synth.EOS, fp16=False)
    arms = {"ours": lambda i: gen.greedy_decode(ours_b[i % len(ours_b)])}
    agree = None
    if stage_ref.available():
        ref_b = [synth.to_device({k: v for k, v in b.items() if not k.startswith("_hero")}, DEV)
                 for b in host]
        ref = reference_generator(model.state_dict())
        arms["reference_bf16_autocast"] = lambda i: ref(ref_b[i % len(ref_b)])
        a, r = gen.greedy_decode(ours_b[0]), ref(ref_b[0])
        first = [sum(1 for x, y in zip(p, q) if x == y) for p, q in zip(a, r)]
        agree = {"captions": len(a), "identical": sum(p == q for p, q in zip(a, r)),
                 "matching_prefix_tokens": first}
    for fn in arms.values():
        events_ms(fn, args.warmup)
    times = {k: [] for k in arms}
    for _ in range(args.repeats):                      # alternate the arms
        for k, fn in arms.items():
            times[k].append(events_ms(fn, args.batches))
    # one decode step of the vocabulary GEMM + argmax at the preset's caption count, against the
    # decode loop's per-step time (batch time less the encoder side, over max_step)
    N = max(n_caps)
    h = torch.randn(N, 768, device=DEV).to(torch.bfloat16)
    flat, w = model._weights(DEV)
    logits = torch.empty(N, w["emb_bf16"].shape[0], device=DEV)
    ids = torch.empty(N, 1, dtype=torch.int32, device=DEV)
    vals = torch.empty(N, 1, device=DEV)

    def lm(i):
        ops.gemm(h, w["emb_bf16"], logits, bias=w["lm_bias"])
        ops.rank_topk(logits, w["n_valid"], 1, vals, ids)
    events_ms(lm, 20)
    lm_ms = events_ms(lm, 500)

    def encode(i):
        with torch.no_grad():
            b = ours_b[i % len(ours_b)]
            y, tplan = model.encode(b)
            tdev = tplan.to(DEV, tplan.decode_arrays(MAX_STEP))
            model._cross_kv(w, model._gather_segments(y, tplan, tdev))
    events_ms(encode, 2)
    enc_ms = events_ms(encode, args.batches)
    ours_ms = sorted(times["ours"])[len(times["ours"]) // 2]
    step_ms = (ours_ms - enc_ms) / MAX_STEP
    out = {"gpu": name, "power_limit": watts,
           "preset": "syn_tvc_val: 8 videos of 20-100 frames, 2-6 caption segments each "
                     "(one empty), max_step 30; 6 + 3 encoder layers, 2 decoder layers, H 768, "
                     "vocabulary 50272",
           "captions_per_batch": n_caps, "batches": args.batches, "warmup": args.warmup,
           "repeats": args.repeats,
           "ms_per_batch": times,
           "ms_per_batch_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
           "greedy_agreement_with_reference_bf16": agree,
           "encode_ms_per_batch": enc_ms, "decode_step_ms": step_ms,
           "dec_attn_us_per_call": {
               "decode_step_self (rows 32, 12 heads, 16 keys)": 1e3 * attn_ms(32, 12, 16, 30),
               "decode_step_self (rows 32, 12 heads, 30 keys)": 1e3 * attn_ms(32, 12, 30, 30),
               "cross (rows 32, 12 heads, 16 keys)": 1e3 * attn_ms(32, 12, 16, 16)},
           "logits_argmax_ms_per_step": lm_ms,
           "logits_argmax_share_of_step": lm_ms / step_ms}
    print(json.dumps(out, indent=1))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
