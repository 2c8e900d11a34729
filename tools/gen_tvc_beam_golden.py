"""Writes tests/golden/tvc_beam_tiny.npz: beam search over the reference's HeroForTvc.decode
(model/tvc.py) on the tiny model and batch of tests/golden/tvc_tiny.npz (same configuration and
seeded weights, tools/gen_tvc_golden.py), in fp32 on the CPU, re-running the whole prefix at every
step.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_tvc_beam_golden.py

The search (`beam_search` below, written for this fixture; the reference decodes greedily only)
follows TvcGenerator.beam_ids: R = captions x B rows, beam 0 of each caption at score 0 and the
others at -inf; a live beam offers its top-B tokens (descending logit, ties to the lower id) at
score + log-probability, a finished beam (one that has emitted EOS) offers EOS at its score; the B
best candidates become the next beams, ties to the lower parent * B + rank; all max_step steps run;
the chosen beam maximises score / len ** alpha, len = tokens up to and including the first EOS.

Stored for B in {1, 3, 5}: `b<B>_steps` [N, T, B, T], the B token histories after every step (-1
past the step); `b<B>_score` / `b<B>_len` [N, B], the final scores and lengths; `b<B>_margin` [N,
T], the smallest score gap at each step that decides which beams are kept (the B-th best candidate
minus the (B+1)-th, and for a selected candidate of rank B - 1 its parent's B-th minus (B+1)-th
logit: below it a perturbation can swap a kept hypothesis for another; the order of the kept beams
does not change the next step's candidates); and for alpha in {0, 1}
`b<B>_a<alpha>_pick` [N] (chosen beam) and `b<B>_a<alpha>_pick_gap` [N] (its normalised score minus
the runner-up's). Checked here: B = 1 cut at EOS equals tvc_tiny.npz's greedy ids cut at EOS.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hero_b200 import synth  # noqa: E402

BEAMS = (1, 3, 5)
ALPHAS = (0, 1)


def beam_search(last_logits, n_cap, beam, max_step, bos, eos, vocab):
    """Torch beam search. `last_logits(ids)` maps the (R, t + 1) input ids (BOS first) to the fp32
    logits (R, >= vocab) of the last position. Returns a dict of numpy arrays: steps [N, T, B, T],
    score / len [N, B], margin [N, T]."""
    R, T = n_cap * beam, max_step
    score = torch.full((R,), float("-inf"))
    score[::beam] = 0.0
    fin = torch.zeros(R, dtype=torch.bool)
    length = torch.zeros(R, dtype=torch.long)
    hist = torch.zeros(R, 0, dtype=torch.long)
    inputs = torch.full((R, 1), bos, dtype=torch.long)
    steps = np.full((n_cap, T, beam, T), -1, np.int64)
    margin = np.full((n_cap, T), np.inf)
    for t in range(T):
        z = last_logits(inputs)[:, :vocab].float()
        lse = torch.logsumexp(z, dim=1)
        k1 = min(beam + 1, vocab)
        order = torch.sort(z, dim=1, descending=True, stable=True).indices[:, :k1]
        top = z.gather(1, order)
        logp = top[:, :beam] - lse[:, None]
        new_rows, new_tok = [], []
        n_score, n_fin, n_len = score.clone(), fin.clone(), length.clone()
        for n in range(n_cap):
            cand = []                               # (score, flat index, parent row, token, rank)
            for p in range(beam):
                r = n * beam + p
                if fin[r]:
                    cand.append((float(score[r]), p * beam, r, eos, 0))
                else:
                    for k in range(beam):
                        cand.append(((score[r] + logp[r, k]).item(), p * beam + k, r,
                                     int(order[r, k]), k))
            cand.sort(key=lambda c: (-c[0], c[1]))
            gaps = [cand[beam - 1][0] - cand[beam][0]] if len(cand) > beam and \
                cand[beam][0] != float("-inf") else []
            for s, _, rp, tok, k in cand[:beam]:
                if not fin[rp] and k == beam - 1 and k1 > beam:
                    gaps.append(float(top[rp, beam - 1] - top[rp, beam]))
            margin[n, t] = min(gaps, default=np.inf)
            for b, (s, _, rp, tok, k) in enumerate(cand[:beam]):
                r = n * beam + b
                n_score[r] = s
                n_fin[r] = bool(fin[rp]) or tok == eos
                n_len[r] = length[rp] if fin[rp] else t + 1
                new_rows.append(rp)
                new_tok.append(tok)
        rows = torch.tensor(new_rows)
        tok = torch.tensor(new_tok)
        hist = torch.cat([hist[rows], tok[:, None]], 1)
        inputs = torch.cat([inputs[rows], tok[:, None]], 1)
        score, fin, length = n_score, n_fin, n_len
        steps[:, t, :, :t + 1] = hist.view(n_cap, beam, t + 1).numpy()
    return {"steps": steps, "score": score.view(n_cap, beam).numpy(),
            "len": length.view(n_cap, beam).numpy(), "margin": margin}


def pick(score, length, alpha):
    """(chosen beam [N], its normalised score minus the runner-up's [N])."""
    norm = score.astype(np.float64) / np.power(length.astype(np.float64), float(alpha))
    best = np.argmax(norm, axis=1)
    srt = -np.sort(-norm, axis=1)
    gap = srt[:, 0] - srt[:, 1] if norm.shape[1] > 1 else np.full(norm.shape[0], np.inf)
    return best, gap


def cut(ids, eos):
    out = []
    for i in ids:
        if i == eos:
            break
        out.append(int(i))
    return out


def reference_last_logits(model, batch, beam):
    """last_logits over the reference's HeroForTvc.decode for `beam` rows per caption."""
    enc = model.encode(batch).repeat_interleave(beam, 0)
    mask = batch["cap_attn_mask"].repeat_interleave(beam, 0)

    def last(ids):
        ids = ids.to(enc.device)
        pos = torch.arange(ids.shape[1], device=enc.device).unsqueeze(0)
        return model.decode(enc, mask, ids, pos, None, compute_loss=False)[:, -1].float().cpu()
    return last


def main():
    import tools.gen_tvc_golden as tg
    from oracle import gen_golden as gg
    gg.install_stubs()
    model, _ = tg.build(0.1)
    tx = np.load(os.path.join(ROOT, "tests", "golden", "tvc_tiny.npz"))
    b = tg.batch("val")
    n_cap = b["cap_attn_mask"].shape[0]
    out = {"max_step": np.int64(tg.MAX_STEP), "beams": np.asarray(BEAMS),
           "alphas": np.asarray(ALPHAS)}
    with torch.no_grad():
        for beam in BEAMS:
            res = beam_search(reference_last_logits(model, tg.batch("val"), beam), n_cap, beam,
                              tg.MAX_STEP, synth.BOS, synth.EOS, tg.VOCAB)
            for k, v in res.items():
                out[f"b{beam}_{k}"] = v
            for a in ALPHAS:
                best, gap = pick(res["score"], res["len"], a)
                out[f"b{beam}_a{a}_pick"] = best
                out[f"b{beam}_a{a}_pick_gap"] = gap
            print(f"B = {beam}: lengths {res['len'][np.arange(n_cap), out[f'b{beam}_a0_pick']]}, "
                  f"steps before the first margin <= 0.1 per caption "
                  f"{[int(np.argmax(np.r_[m, 0.0] <= 0.1)) for m in res['margin']]}")
    final = out["b1_steps"][:, -1, 0]
    for r in range(n_cap):
        assert cut(final[r], synth.EOS) == cut(tx["greedy_ids"][r], synth.EOS), r
    print("B = 1 cut at EOS == tvc_tiny.npz greedy ids cut at EOS")
    dst = os.path.join(ROOT, "tests", "golden", "tvc_beam_tiny.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}")


if __name__ == "__main__":
    main()
