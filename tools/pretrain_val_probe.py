"""Pretraining validation on one GPU at real dimensions (6 + 3 layers, H 768, vocabulary 50 272,
4352-d features) on SYN-HT100M-dense batches of 8 clips: per task, ms per validation batch of
evalpass.validate_<task> (plans attached on the host, two arms alternated with the reference
when it can run), the peak device memory of one MLM and one MFM-NCE batch, and the error of the
fused MLM / MFM-NCE losses against the model's own fp32 torch logits next to that of the same
logits under bf16 autocast. The card's name and power limit name the output file
(tools/pretrain_val_probe_<card>_<watts>w.json).

The reference arm runs pretrain.py's own validate functions under bf16 autocast on the staged
reference model; it needs pretrain.py (HERO_REFERENCE=<checkout>), which oracle/stage_ref.py does
not stage, and is recorded as skipped without it.

    python tools/pretrain_val_probe.py [--out-dir tools]
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

from hero_b200 import evalpass, synth  # noqa: E402
from hero_b200.plan import attach_plan  # noqa: E402
from oracle import gen_golden as gg  # noqa: E402
from oracle import stage_ref  # noqa: E402
from tests import pretrain_val_batches as pv  # noqa: E402
from tools.videoqa_probe import card, events_ms  # noqa: E402

DEV = torch.device("cuda")
FNS = {"mlm": evalpass.validate_mlm, "mffr": evalpass.validate_mffr,
       "mfm-nce": evalpass.validate_mfm_nce, "fom": evalpass.validate_fom,
       "vsm": lambda m, loader: evalpass.validate_vsm(m, loader, pv.Opts)}


def file_name(name, watts):
    model = re.search(r"[A-Z]\d{2,4}", name)
    w = int(round(float(re.sub(r"[^0-9.]", "", watts))))
    return f"pretrain_val_probe_{(model.group(0) if model else 'gpu').lower()}_{w}w.json"


def device_batches(task, n, attach):
    out = []
    for i in range(n):
        b = pv.real_batch(task, i)
        if attach:
            if task == "mlm":
                evalpass.attach_mlm_plan(b)
            else:
                attach_plan(b, "vsm" if task == "vsm" else "repr")
        out.append(synth.to_device(b, DEV))
    return out


def reference_arms(model, n):
    """pretrain.py's validate functions on the reference model (same weights) under bf16
    autocast, or None when pretrain.py cannot be imported."""
    ref_root = os.environ.get("HERO_REFERENCE")
    if not ref_root or not os.path.isfile(os.path.join(ref_root, "pretrain.py")) or \
            stage_ref.available() is None:
        return None
    gg.REF = ref_root
    gg.install_stubs()
    import pretrain
    from model.model import VideoModelConfig as RefConfig
    from model.pretrain import HeroForPretraining as RefModel
    pretrain.all_gather_list = lambda x: [x]
    j = gg.model_json(768, 3072, 12, 6, 3, pv.REAL_VOCAB)
    j["q_config"] = dict(j["c_config"], num_hidden_layers=1)
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(j, f)
        path = f.name
    ref = RefModel(RefConfig(path), vfeat_dim=pv.REAL_VFEAT, max_frm_seq_len=100,
                   **pv.LOSS_WEIGHTS)
    os.unlink(path)
    ref.load_state_dict(model.state_dict(), strict=False)
    ref = ref.to(DEV).eval()
    fns = {"mlm": pretrain.validate_mlm, "mffr": pretrain.validate_mffr,
           "mfm-nce": pretrain.validate_mfm_nce, "fom": pretrain.validate_fom,
           "vsm": lambda m, loader: pretrain.validate_vsm(m, loader, pv.Opts)}

    def arm(task):
        batches = device_batches(task, n, False)

        def run(i):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                fns[task](ref, [dict(b) for b in batches])
        return run
    return {t: arm(t) for t in pv.TASKS}


def peak_mb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn(0)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def errors(model):
    """|validate_<task> loss - fp32 torch| against |bf16-autocast torch - fp32 torch|, per row."""
    out = {}
    for task in ("mlm", "mfm-nce"):
        batches = [synth.to_device(pv.real_batch(task, i), DEV) for i in range(2)]
        l32, h32, n, gap = pv.torch_logit_metrics(model, task, batches)
        lac, hac, _, _ = pv.torch_logit_metrics(model, task, batches, autocast=True)
        got = FNS[task](model, batches)
        out[task] = {"rows": n, "fp32_loss": l32 / n, "fused_loss": got["loss"],
                     "autocast_loss": lac / n,
                     "fused_abs_err": abs(got["loss"] - l32 / n),
                     "autocast_abs_err": abs(lac - l32) / n,
                     "fp32_hits": h32, "fused_hits": round(got["acc"] * n), "autocast_hits": hac,
                     "rows_with_gap_below_1e-2": int((gap < 1e-2).sum())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "tools"))
    args = ap.parse_args()
    name, watts = card()
    model = pv.real_model(DEV)
    n = args.batches
    loaders = {t: device_batches(t, n, True) for t in pv.TASKS}
    arms = {t: {"ours": (lambda t: lambda i: FNS[t](model, loaders[t]))(t)} for t in pv.TASKS}
    ref = reference_arms(model, n)
    if ref is not None:
        for t in pv.TASKS:
            arms[t]["reference_bf16_autocast"] = ref[t]
    times = {t: {k: [] for k in a} for t, a in arms.items()}
    for t, a in arms.items():
        for fn in a.values():
            for i in range(args.warmup):                 # library load, caches
                fn(i)
        for _ in range(args.repeats):                    # alternate the arms
            for k, fn in a.items():
                times[t][k].append(events_ms(fn, 1) / n)
    peaks = {t: {k: peak_mb(lambda i, t=t, fn=fn: fn(i)) for k, fn in arms[t].items()}
             for t in ("mlm", "mfm-nce")}
    out = {"gpu": name, "power_limit": watts,
           "preset": "SYN-HT100M-dense, 8 clips per batch (30 frames, 6 subtitles of 5 frames + "
                     "20 tokens); 6 + 3 layers, H 768, vocabulary 50272, 4352-d features",
           "batches_per_pass": n, "repeats": args.repeats,
           "reference": "pretrain.py validate functions under bf16 autocast" if ref is not None
           else "skipped: pretrain.py is not available (oracle/stage_ref.py stages the "
                "reference's packages only; set HERO_REFERENCE)",
           "ms_per_batch": times,
           "ms_per_batch_median": {t: {k: sorted(v)[len(v) // 2] for k, v in a.items()}
                                   for t, a in times.items()},
           "peak_mb_per_pass": peaks,
           "loss_error_vs_fp32_logits": errors(model)}
    print(json.dumps(out, indent=1))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, file_name(name, watts)), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
