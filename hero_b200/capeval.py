"""TVC caption metrics on the GPU: BLEU-1..4, ROUGE-L and CIDEr-D of decoded captions, equal to the
COCO caption scorers the reference's eval/tvc.py:TVCEval calls (eval/pycocoevalcap/{bleu,rouge,
cider}), without Java.

`TVCEval(ref_path)(records)` scores the records of `evalpass.decode_tvc` (or of the reference's
`decode`) against an annotation file, as the reference does, and returns
{"Bleu_1", "Bleu_2", "Bleu_3", "Bleu_4", "ROUGE_L", "CIDEr"}, each x 100. There is no "METEOR": the
reference's METEOR is a Java jar with WordNet and paraphrase tables, and is not restated here.

The reference tokenizes with Stanford CoreNLP's PTBTokenizer (Java). `ptb_tokenize` restates the
part of it that captions use; `tokenize=None` takes text that is already tokenized (for instance the
Java tokenizer's output, which then gives the reference's exact numbers).

`caption_scores(hyps, refs)` is the layer underneath: token lists in, corpus scores and per-clip
arrays out. Words become ids through one vocabulary per call, the sentences go to the device in one
upload, the kernels of csrc/capeval.cu produce per-clip integers and fp64 partials, and one copy
brings them back. The host finishes in the reference's expression order: BLEU in Python floats,
ROUGE-L and the means in numpy, so BLEU and ROUGE-L are bit-equal to the reference and CIDEr-D
agrees to fp64 rounding (its sums run in another order).
"""
import json
import math
import re

import numpy as np
import torch

from . import ops

BLEU_TINY, BLEU_SMALL = 1e-15, 1e-9        # bleu_scorer.py compute_score
ROUGE_BETA = 1.2
METRICS = ("Bleu_1", "Bleu_2", "Bleu_3", "Bleu_4", "ROUGE_L", "CIDEr")

# ---------------------------------------------------------------------------------------------
# Tokenizer: Stanford PTBTokenizer -preserveLines -lowerCase, then the reference's punctuation
# filter. Brackets are dropped outright: PTBTokenizer writes them as -LRB- / -RRB- / -LCB- / -RCB-,
# which the filter removes (assuming -lowerCase leaves those escapes upper-case).
_DROP = frozenset(["''", "'", "``", "`", '"', ".", "?", "!", ",", ":", "-", "--", "...", ";",
                   "(", ")", "[", "]", "{", "}", "-lrb-", "-rrb-", "-lcb-", "-rcb-"])
_LEAD = "\"'`([{"
_TRAIL = ".,;:?!\"'`)]}"
# Abbreviations that keep their period (PTBTokenizer's list is longer; these are the ones captions
# meet). Letter-dot acronyms such as "u.s." or "a.m." also stay whole.
ABBREVIATIONS = frozenset(["mr.", "mrs.", "ms.", "dr.", "prof.", "st.", "jr.", "sr.", "vs.",
                           "etc.", "no.", "mt.", "ft.", "inc.", "co.", "ltd.", "jan.", "feb.",
                           "aug.", "sept.", "oct.", "nov.", "dec."])
_ACRONYM = re.compile(r"^(?:[a-z]\.){2,}$")
_CLITIC = re.compile(r"^(.+?)('s|'re|'ve|'ll|'d|'m)$")
_SPLIT_WORDS = {"cannot": ["can", "not"], "gonna": ["gon", "na"], "gotta": ["got", "ta"],
                "wanna": ["wan", "na"]}


def _word_tokens(w):
    """One whitespace-free chunk without its leading / trailing punctuation."""
    if w in _SPLIT_WORDS:
        return _SPLIT_WORDS[w]
    if len(w) > 3 and w.endswith("n't"):
        return [w[:-3], "n't"]
    m = _CLITIC.match(w)
    if m:
        return [m.group(1), m.group(2)]
    return [w]


def _chunk_tokens(chunk):
    lead, trail = [], []
    while chunk and chunk[0] in _LEAD and chunk not in ("'s", "'re", "'ve", "'ll", "'d", "'m"):
        lead.append(chunk[0])
        chunk = chunk[1:]
    while chunk:
        if chunk.endswith("..."):
            trail.append("...")
            chunk = chunk[:-3]
        elif chunk[-1] in _TRAIL:
            if chunk[-1] == "." and (chunk in ABBREVIATIONS or _ACRONYM.match(chunk)):
                break
            if chunk[-1] == "'" and chunk.endswith("n'"):    # "goin'" keeps its apostrophe
                break
            trail.append(chunk[-1])
            chunk = chunk[:-1]
        else:
            break
    core = _word_tokens(chunk) if chunk else []
    return lead + core + trail[::-1]


def ptb_tokenize(text):
    """Caption text -> space-separated lower-case tokens with punctuation removed, as the
    reference's PTBTokenizer wrapper returns them: `.` `,` `;` `:` `?` `!` `...`, quotes and
    brackets are split off and dropped; the clitics 's 're 've 'll 'd 'm n't become tokens
    ("don't" -> "do n't", "can't" -> "ca n't"); "cannot", "gonna", "gotta", "wanna" -> "can not",
    "gon na", "got ta", "wan na"; hyphenated words and numbers such as 3.5 or 1,000 stay whole, and
    so do the ABBREVIATIONS and letter-dot acronyms ("u.s.")."""
    out = []
    for chunk in text.lower().split():
        out.extend(t for t in _chunk_tokens(chunk) if t not in _DROP)
    return " ".join(out)


# ---------------------------------------------------------------------------------------------
# Device pass and host finish.
class CaptionPack:
    """Host side of one scoring call: the vocabulary-encoded CSR arrays and every size the
    launches need, all known before anything reaches the device."""

    def __init__(self, hyps, refs):
        n_clips = len(hyps)
        if n_clips == 0 or len(refs) != n_clips:
            raise ValueError(f"caption_scores: {n_clips} hypotheses and {len(refs)} reference "
                             "lists; need one list per hypothesis and at least one clip")
        n_refs = np.fromiter(map(len, refs), np.int64, n_clips)
        if (n_refs == 0).any():
            raise ValueError(f"caption_scores: clip {int(np.argmin(n_refs))} has no reference")
        sents = list(hyps)
        for r in refs:
            sents.extend(r)
        lens = np.fromiter(map(len, sents), np.int64, len(sents))
        if lens.max() > ops.CAPTION_MAX_LEN:
            s = int(np.argmax(lens))
            what = f"hypothesis {s}" if s < n_clips else f"a reference of clip " \
                f"{int(np.searchsorted(np.cumsum(n_refs), s - n_clips, side='right'))}"
            raise ValueError(f"caption_scores: {what} has {int(lens[s])} words; at most "
                             f"{ops.CAPTION_MAX_LEN} are supported")
        vocab = {}
        tok = np.fromiter((vocab.setdefault(w, len(vocab) + 1) for s in sents for w in s),
                          np.int64, int(lens.sum()))
        if len(vocab) > ops.CAPTION_MAX_WORD:
            raise ValueError(f"caption_scores: {len(vocab)} distinct words; at most "
                             f"{ops.CAPTION_MAX_WORD} are supported")
        grams = sum(np.maximum(0, lens - n + 1) for n in range(1, 5))
        self.sent_off = np.concatenate([[0], np.cumsum(lens)])
        self.gram_off = np.concatenate([[0], np.cumsum(grams)])
        if max(self.sent_off[-1], self.gram_off[-1]) >= 2 ** 31:
            raise ValueError(f"caption_scores: {int(self.sent_off[-1])} words / "
                             f"{int(self.gram_off[-1])} n-grams; at most 2^31 - 1 are supported")
        self.ref_off = np.concatenate([[0], np.cumsum(n_refs)])
        self.tok = tok
        self.lens, self.n_refs, self.n_clips = lens, n_refs, n_clips
        self.vocab_size = len(vocab)
        self.n_grams = int(self.gram_off[-1])
        self.n_ref_grams = int(self.gram_off[-1] - self.gram_off[n_clips])
        self.max_hyp_grams = int(grams[:n_clips].max())
        # idf = log(n_clips) - log(max(1, df)): the host's logs (np.log, as cider_scorer.py takes
        # them), so an n-gram in every clip's references gets exactly 0
        self.log_n = np.array([0.0] + [np.log(float(d)) for d in range(1, n_clips + 1)])

    def upload(self, device):
        """One host-to-device copy of log_n (fp64) and the int32 CSR arrays; returns the device
        views (sent_off, gram_off, ref_off, tok, log_n)."""
        parts = [self.log_n.view(np.int32), self.sent_off, self.gram_off, self.ref_off, self.tok]
        sizes = [p.size for p in parts]
        host = torch.empty(sum(sizes), dtype=torch.int32, pin_memory=device.type == "cuda")
        hv = host.numpy()
        o = 0
        for p, n in zip(parts, sizes):
            hv[o:o + n] = p
            o += n
        flat = host.to(device, non_blocking=True)
        self._host = host            # pinned memory stays alive until the copy has been consumed
        views, o = [], 0
        for n in sizes:
            views.append(flat[o:o + n])
            o += n
        return views[1], views[2], views[3], views[4], views[0].view(torch.float64)


def _device():
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() \
        else torch.device("cpu")


def device_stats(pack, device=None):
    """The device pass of one CaptionPack: upload and kernels, no host synchronisation. Returns
    the fp64 device tensor of ops.caption_stats."""
    sent_off, gram_off, ref_off, tok, log_n = pack.upload(device or _device())
    return ops.caption_stats(sent_off, gram_off, ref_off, tok, log_n, n_grams=pack.n_grams,
                             n_ref_grams=pack.n_ref_grams, max_hyp_grams=pack.max_hyp_grams)


def finish(pack, out):
    """Corpus scores and per-clip arrays from the returned counts (numpy fp64 [5 C + 5 R]), in
    the expression order of bleu_scorer.py, rouge.py and cider_scorer.py."""
    C = pack.n_clips
    clip = out[:5 * C].reshape(C, 5)
    ref = out[5 * C:].reshape(-1, 5)
    correct = clip[:, :4].astype(np.int64)
    reflen = clip[:, 4].astype(np.int64)
    testlen = pack.lens[:C]
    guess = np.stack([np.maximum(0, testlen - k) for k in range(4)], 1)

    # BLEU (option 'closest'), per clip and from the summed integers, in Python floats
    bleu_list = [[] for _ in range(4)]
    for tl, rl, cc, gg in zip(testlen.tolist(), reflen.tolist(), correct.tolist(), guess.tolist()):
        b = 1.
        for k in range(4):
            b *= (float(cc[k]) + BLEU_TINY) / (float(gg[k]) + BLEU_SMALL)
            bleu_list[k].append(b ** (1. / (k + 1)))
        ratio = (tl + BLEU_TINY) / (rl + BLEU_SMALL)
        if ratio < 1:
            for k in range(4):
                bleu_list[k][-1] *= math.exp(1 - 1 / ratio)
    tot_c, tot_g = correct.sum(0).tolist(), guess.sum(0).tolist()
    tot_t, tot_r = int(testlen.sum()), int(reflen.sum())
    bleus, b = [], 1.
    for k in range(4):
        b *= float(tot_c[k] + BLEU_TINY) / (tot_g[k] + BLEU_SMALL)
        bleus.append(b ** (1. / (k + 1)))
    ratio = (tot_t + BLEU_TINY) / (tot_r + BLEU_SMALL)
    if ratio < 1:
        for k in range(4):
            bleus[k] *= math.exp(1 - 1 / ratio)

    # ROUGE-L. rouge.py splits on " ", so an empty sentence is one empty token, which matches only
    # another empty sentence.
    hl = np.repeat(testlen, pack.n_refs)
    rl = pack.lens[C:]
    lcs = np.where((hl == 0) & (rl == 0), 1, ref[:, 4].astype(np.int64))
    prec = lcs / np.maximum(hl, 1).astype(np.float64)
    rec = lcs / np.maximum(rl, 1).astype(np.float64)
    starts = pack.ref_off[:-1]
    pm, rm = np.maximum.reduceat(prec, starts), np.maximum.reduceat(rec, starts)
    b2 = ROUGE_BETA ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        rouge = np.where((pm != 0) & (rm != 0), ((1 + b2) * pm * rm) / (rm + b2 * pm), 0.0)

    # CIDEr-D: similarities summed over the references, mean over n, / references, x 10
    cider = np.add.reduceat(ref[:, :4], starts, axis=0).mean(axis=1) / pack.n_refs * 10.0

    scores = {"Bleu_1": bleus[0], "Bleu_2": bleus[1], "Bleu_3": bleus[2], "Bleu_4": bleus[3],
              "ROUGE_L": np.mean(rouge), "CIDEr": np.mean(cider)}
    per_clip = {"bleu": np.array(bleu_list).T, "correct": correct, "guess": guess,
                "testlen": testlen, "reflen": reflen, "rouge_l": rouge, "cider": cider}
    return scores, per_clip


def caption_scores(hyps, refs):
    """hyps: one token list per clip; refs: per clip a non-empty list of token lists (at most 1024
    tokens per sentence, 65 535 distinct tokens per call; ValueError otherwise, before any launch).
    Returns (scores, per_clip): scores {"Bleu_1".."Bleu_4", "ROUGE_L", "CIDEr"} as the COCO scorers'
    compute_score returns them (not x 100); per_clip "bleu" [C, 4], BLEU "correct" / "guess"
    [C, 4], "testlen" / "reflen" [C] (closest reference length), "rouge_l" [C], "cider" [C]."""
    pack = CaptionPack(hyps, refs)
    out = device_stats(pack).cpu().numpy()
    return finish(pack, out)


def _remove_nonascii(text):
    return "".join(ch if ord(ch) < 128 else " " for ch in text)


class TVCEval:
    """Drop-in for the reference's eval/tvc.py:TVCEval without METEOR (a Java jar, not restated):
    references are read once from the annotation file (JSON lines with 'clip_id' and 'descs'), and
    each call scores a list of result records {'clip_id', 'descs': [{'desc': caption}, ...]}.
    Text is strip()ped, non-ASCII characters become spaces, and `tokenize` (ptb_tokenize; None:
    the text is already tokenized) produces space-separated tokens."""

    def __init__(self, ref_path, tokenize=ptb_tokenize):
        self.tokenize = tokenize
        self.id2refs = {}
        with open(ref_path) as f:
            for ex in map(json.loads, f):
                self.id2refs[ex["clip_id"]] = [self._tokens(cap["desc"]) for cap in ex["descs"]]

    def _tokens(self, text):
        text = _remove_nonascii(text.strip())
        return (self.tokenize(text) if self.tokenize is not None else text).split()

    def __call__(self, json_res):
        """Corpus BLEU-1..4, ROUGE-L and CIDEr-D x 100 of the records' first captions; a later
        record with the same clip_id replaces an earlier one."""
        id2hyp = {res["clip_id"]: res["descs"][0]["desc"] for res in json_res}
        if id2hyp.keys() != self.id2refs.keys():
            missing = [c for c in self.id2refs if c not in id2hyp]
            extra = [c for c in id2hyp if c not in self.id2refs]
            raise ValueError(f"TVCEval: the results must cover exactly the annotated clips; "
                             f"missing {missing}, extra {extra}")
        clips = list(self.id2refs)
        scores, _ = caption_scores([self._tokens(id2hyp[c]) for c in clips],
                                   [self.id2refs[c] for c in clips])
        return {k: scores[k] * 100 for k in METRICS}
