"""TEST INFRASTRUCTURE: a plain restatement of ops.caption_stats (hero_caption_ngrams, the df sort
and hero_caption_clip_stats; include/hero_b200.h, csrc/capeval.cu), written from its contract, so
capeval runs on a CPU-only box and the kernels have a reference on the GPU. N-grams are word-id
tuples in Counters, df counts the clips whose references contain a tuple, and the LCS is the
textbook dynamic programme, one row per reference word (numpy running maximum)."""
from collections import Counter

import numpy as np
import torch


def _ngrams(words):
    c = Counter()
    for n in range(1, 5):
        for i in range(len(words) - n + 1):
            c[words[i:i + n]] += 1
    return c


def _lcs(a, b):
    a = np.asarray(a)
    row = np.zeros(len(a) + 1, dtype=np.int64)
    for w in b:
        t = row.copy()
        t[1:] = np.maximum(row[1:], row[:-1] + (a == w))
        row = np.maximum.accumulate(t)
    return int(row[-1])


def clip_stats(sents, ref_off, log_n):
    """sents: word-id tuples, the C hypotheses then the references -> fp64 [5 C + 5 R]."""
    C = len(ref_off) - 1
    counts = [_ngrams(s) for s in sents]
    df = Counter()
    for c in range(C):
        df.update(set().union(*(counts[C + j] for j in range(ref_off[c], ref_off[c + 1]))))
    ref_len = log_n[C]

    def vec(cnt):
        w = {g: k * (ref_len - log_n[max(1, df[g])]) for g, k in cnt.items()}
        norm = [np.sqrt(sum(v * v for g, v in w.items() if len(g) == n)) for n in range(1, 5)]
        return w, norm

    out = np.zeros(5 * len(sents))
    for c in range(C):
        hyp, hc = sents[c], counts[c]
        refs = list(range(C + ref_off[c], C + ref_off[c + 1]))
        for n in range(1, 5):
            out[5 * c + n - 1] = sum(min(k, max(counts[r][g] for r in refs))
                                     for g, k in hc.items() if len(g) == n)
        out[5 * c + 4] = min((abs(len(sents[r]) - len(hyp)), len(sents[r])) for r in refs)[1]
        wh, nh = vec(hc)
        for r in refs:
            wr, nr = vec(counts[r])
            delta = float(max(0, len(hyp) - 1) - max(0, len(sents[r]) - 1))
            o = 5 * r                      # the references follow the 5 C clip entries
            for n in range(1, 5):
                val = sum(min(v, wr.get(g, 0.0)) * wr.get(g, 0.0)
                          for g, v in wh.items() if len(g) == n)
                if nh[n - 1] != 0 and nr[n - 1] != 0:
                    val /= nh[n - 1] * nr[n - 1]
                out[o + n - 1] = val * np.exp(-(delta ** 2) / 72.0)
            out[o + 4] = _lcs(hyp, sents[r])
    return out


def caption_stats(sent_off, gram_off, ref_off, tok, log_n, *, n_grams, n_ref_grams,
                  max_hyp_grams):
    so, tk = sent_off.cpu().numpy(), tok.cpu().numpy()
    sents = [tuple(int(w) for w in tk[so[s]:so[s + 1]]) for s in range(len(so) - 1)]
    go = gram_off.cpu().numpy()
    assert n_grams == go[-1] and n_ref_grams == go[-1] - go[len(ref_off) - 1]
    assert max_hyp_grams == (go[1:len(ref_off)] - go[:len(ref_off) - 1]).max()
    out = clip_stats(sents, ref_off.cpu().numpy(), log_n.cpu().numpy())
    return torch.from_numpy(out).to(tok.device)


def install(monkeypatch):
    from hero_b200 import ops
    monkeypatch.setattr(ops, "caption_stats", caption_stats)
