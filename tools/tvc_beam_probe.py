"""TVC beam search on one GPU: ms per batch of TvcGenerator.greedy_decode and beam_search (B = 3
and 5) on syn_tvc_val (8 videos, 2-6 caption segments each, max_step 30) at real dimensions (6 + 3
encoder layers, 2 decoder layers, H 768, vocabulary 50 272), against the same beam search written
in torch over the reference's HeroForTvc.decode (staged under oracle/_ref) under bf16 autocast,
which re-runs the whole prefix at every step and selects on the host (the yardstick), the arms
alternated; each new kernel's time per launch back to back (host enqueue included) and its own
device time from torch.profiler, taken in a child process with HERO_SERIAL_PROFILE=1 (with
programmatic dependent launch a kernel's recorded duration would include its wait on the one
before it); beam_logprob_topk's device time over B at a fixed row count against the HBM bound of
its one read; and the share of a beam step spent in the vocabulary GEMM + beam_logprob_topk. The card's name and power limit are read in the same run and
name the output file (tools/tvc_beam_probe_<card>_<watts>w.json).

    python tools/tvc_beam_probe.py [--out-dir tools]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import ops, synth  # noqa: E402
from hero_b200.model import VideoModelConfig  # noqa: E402
from hero_b200.plan import attach_plan  # noqa: E402
from hero_b200.tvc import HeroForTvc, TvcGenerator, _beam_state  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import stage_ref  # noqa: E402
from tools import gen_tvc_beam_golden as gb  # noqa: E402
from tools.tvc_probe import config_path  # noqa: E402
from tools.videoqa_probe import card, events_ms  # noqa: E402

DEV = torch.device("cuda")
MAX_STEP = 30
BEAMS = (3, 5)
HBM_TB_S = 3.35          # H100 SXM data sheet HBM3 bandwidth


def device_us(fn, match, n=200):
    """Mean device time per launch (us) of the kernels whose name contains `match`, from the
    kernel durations torch.profiler records over n launches of fn (no host enqueue in it)."""
    fn(0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(n):
            fn(i)
        torch.cuda.synchronize()
    d = [e.time_range.elapsed_us() for e in prof.events()
         if e.device_type == torch.autograd.DeviceType.CUDA and match in e.name]
    return sum(d) / len(d)


def topk_sweep(n, V, rows):
    """beam_logprob_topk device time over B at `rows` rows of the vocabulary logits (n of V
    columns), with the HBM bound of reading them once."""
    logits = torch.randn(rows, V, device=DEV)
    bound_us = rows * n * 4 / (HBM_TB_S * 1e12) * 1e6
    out = {"rows": rows, "hbm_bound_us": bound_us}
    for beam in (1, 3, 4, 5, 8, 16):
        lse = torch.empty(rows, device=DEV)
        logp = torch.empty(rows, beam, device=DEV)
        cols = torch.empty(rows, beam, dtype=torch.int32, device=DEV)
        us = device_us(lambda i: ops.beam_logprob_topk(logits, n, beam, lse, logp, cols),
                       "beam_logprob_topk")
        out[f"b{beam}"] = {"device_us": us, "share_of_hbm_bound": bound_us / us}
    return out


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"tvc_beam_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def reference_beam(state_dict, beam, n_valid):
    gg.REF = stage_ref.available()
    gg.install_stubs()
    from model.model import VideoModelConfig as RefConfig
    from model.tvc import HeroForTvc as RefTvc
    ref = RefTvc(RefConfig(config_path()), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(state_dict)
    ref = ref.to(DEV).eval()

    def run(b):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            n_cap = b["cap_attn_mask"].shape[0]
            return gb.beam_search(gb.reference_last_logits(ref, dict(b), beam), n_cap, beam,
                                  MAX_STEP, synth.BOS, synth.EOS, n_valid)
    return run


def kernel_us(w, n_cap, beam):
    """Per-launch times of the three new kernels at this preset's row count (events over
    back-to-back launches) and their device times (torch.profiler); with `w` (the model's
    weights) also the vocabulary GEMM + beam_logprob_topk per step."""
    R, T, H, V = n_cap * beam, MAX_STEP, 768, w["emb_bf16"].shape[0]
    logits = torch.randn(R, V, device=DEV)
    lse = torch.empty(R, device=DEV)
    logp = torch.empty(R, beam, device=DEV)
    cols = torch.empty(R, beam, dtype=torch.int32, device=DEV)
    out = {}
    fn = lambda i: ops.beam_logprob_topk(logits, w["n_valid"], beam, lse, logp, cols)  # noqa
    events_ms(fn, 20)
    out["beam_logprob_topk"] = 1e3 * events_ms(fn, 500)
    dev = {"beam_logprob_topk": device_us(fn, "beam_logprob_topk")}
    ops.beam_logprob_topk(logits, w["n_valid"], beam, lse, logp, cols)
    slabs = [torch.zeros(R * T + 3 * R, dtype=torch.int32, device=DEV) for _ in range(2)]
    ancs = [torch.zeros(R * T, dtype=torch.int32, device=DEV) for _ in range(2)]
    ids = torch.empty(R, dtype=torch.int32, device=DEV)
    fn = lambda i: ops.beam_select(logp, cols, _beam_state(slabs[0], R, T), ancs[0],  # noqa
                                   _beam_state(slabs[1], R, T), ancs[1], ids, beam=beam,
                                   step=T - 1, max_step=T, eos=synth.EOS)
    events_ms(fn, 20)
    out["beam_select (last step)"] = 1e3 * events_ms(fn, 500)
    dev["beam_select (last step)"] = device_us(fn, "beam_select")
    cache = torch.randn(T * R, 3 * H, device=DEV).to(torch.bfloat16)
    ctx = torch.empty(R, H, dtype=torch.bfloat16, device=DEV)
    for keys in (16, 30):
        idx = torch.randint(0, T * R, (R, T), dtype=torch.int32, device=DEV)
        ln = torch.full((R,), keys, dtype=torch.int32, device=DEV)
        fn = lambda i: ops.dec_attn_gather_fwd(cache[:R, :H], cache[:, H:2 * H],  # noqa
                                               cache[:, 2 * H:], idx, ln, ctx, heads=12,
                                               max_kv_len=keys)
        events_ms(fn, 20)
        out[f"dec_attn_gather_fwd ({keys} keys)"] = 1e3 * events_ms(fn, 1000)
        dev[f"dec_attn_gather_fwd ({keys} keys)"] = device_us(fn, "dec_attn_fwd_kernel")
    if "lm_bias" not in w:
        return out, dev, None
    h = torch.randn(R, H, device=DEV).to(torch.bfloat16)

    def lm(i):
        ops.gemm(h, w["emb_bf16"], logits, bias=w["lm_bias"])
        ops.beam_logprob_topk(logits, w["n_valid"], beam, lse, logp, cols)
    events_ms(lm, 20)
    return out, dev, events_ms(lm, 500)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    ap.add_argument("--device-times", type=int, default=0,
                    help="(child process) print the kernels' device times at this caption count")
    ap.add_argument("--n-valid", type=int, default=50272)
    ap.add_argument("--vocab", type=int, default=50272)
    args = ap.parse_args()
    if args.device_times:
        w = {"n_valid": args.n_valid, "emb_bf16": torch.empty(args.vocab, 1)}
        N = args.device_times
        res = {f"b{beam}": kernel_us(w, N, beam)[1] for beam in BEAMS}
        res["sweep"] = topk_sweep(args.n_valid, args.vocab, N * max(BEAMS))
        print(json.dumps(res))
        return
    name, watts = card()
    torch.manual_seed(0)
    model = HeroForTvc(VideoModelConfig(config_path()), 4352, 100).to(DEV).eval()
    host = [attach_plan(synth.syn_tvc_val(seed=s)) for s in range(args.batches)]
    n_caps = [len(b["clip_ids"]) for b in host]
    ours_b = [synth.to_device(b, DEV) for b in host]
    gen = TvcGenerator(model, MAX_STEP, synth.BOS, synth.EOS, fp16=False)
    flat, w = model._weights(DEV)
    arms = {"greedy_decode": lambda i: gen.greedy_decode(ours_b[i % len(ours_b)])}
    for beam in BEAMS:
        arms[f"beam_search_b{beam}"] = \
            lambda i, beam=beam: gen.beam_search(ours_b[i % len(ours_b)], beam)
    if stage_ref.available():
        ref_b = [synth.to_device({k: v for k, v in b.items() if not k.startswith("_hero")}, DEV)
                 for b in host]
        for beam in BEAMS:
            ref = reference_beam(model.state_dict(), beam, w["n_valid"])
            arms[f"reference_torch_beam_b{beam}_bf16_autocast"] = \
                lambda i, ref=ref: ref(ref_b[i % len(ref_b)])
    for fn in arms.values():
        for i in range(args.warmup):
            fn(i)
    times = {k: [] for k in arms}
    for _ in range(args.repeats):                      # alternate the arms
        for k, fn in arms.items():
            times[k].append(events_ms(fn, args.batches))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}

    def encode(i):
        with torch.no_grad():
            b = ours_b[i % len(ours_b)]
            y, tplan = model.encode(b)
            tdev = tplan.to(DEV, tplan.beam_arrays(MAX_STEP, 5))
            model._cross_kv(w, model._gather_segments(y, tplan, tdev))
    events_ms(encode, 2)
    enc_ms = events_ms(encode, args.batches)
    per_beam = {}
    N = max(n_caps)
    env = dict(os.environ, HERO_SERIAL_PROFILE="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--device-times", str(N),
                        "--n-valid", str(w["n_valid"]), "--vocab", str(w["emb_bf16"].shape[0])],
                       env=env, capture_output=True, text=True, check=True)
    serial = json.loads(r.stdout.strip().splitlines()[-1])
    for beam in BEAMS:
        k_us, _, lm_ms = kernel_us(w, N, beam)
        step_ms = (med[f"beam_search_b{beam}"] - enc_ms) / MAX_STEP
        per_beam[f"b{beam}"] = {"rows": N * beam, "kernel_us_per_launch": k_us,
                                "kernel_device_us": serial[f"b{beam}"],
                                "beam_step_ms": step_ms,
                                "vocab_gemm_plus_logprob_topk_ms": lm_ms,
                                "vocab_gemm_plus_logprob_topk_share_of_step": lm_ms / step_ms}
    out = {"gpu": name, "power_limit": watts,
           "preset": "syn_tvc_val: 8 videos of 20-100 frames, 2-6 caption segments each "
                     "(one empty), max_step 30; 6 + 3 encoder layers, 2 decoder layers, H 768, "
                     "vocabulary 50272",
           "yardstick": "tools/gen_tvc_beam_golden.beam_search over the reference's "
                        "HeroForTvc.decode under bf16 autocast: whole prefix re-run every step, "
                        "selection on the host",
           "captions_per_batch": n_caps, "batches": args.batches, "warmup": args.warmup,
           "repeats": args.repeats, "ms_per_batch": times, "ms_per_batch_median": med,
           "encode_ms_per_batch": enc_ms, "per_beam": per_beam,
           "beam_logprob_topk_over_beam": serial["sweep"]}
    print(json.dumps(out, indent=1))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
