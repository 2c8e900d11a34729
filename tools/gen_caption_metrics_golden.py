"""Writes tests/golden/caption_metrics_tiny.npz: the reference's COCO caption scorers (BLEU-4,
ROUGE-L, CIDEr-D; eval/pycocoevalcap, pure Python) on a seeded, pre-tokenized corpus, and the
reference's eval/tvc.py:TVCEval record flow on it.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python tools/gen_caption_metrics_golden.py

The corpus (space-joined tokens) has empty hypotheses and references, one-word sentences, a tie for
the closest reference length, repeated n-grams that clipping caps, a hypothesis equal to one of its
references, a word in every clip's references (idf 0) and a hypothesis made of it alone, and a
hypothesis of 1024 words. A second, one-clip corpus has ref_len = log(1) = 0. Stored: "corpus" /
"one_clip" (JSON {"hyps": [str], "refs": [[str]]}), per corpus prefix "main." / "one.": "bleu"
[C, 4] (per-clip BLEU-n), "correct" [C, 4] and "reflen" [C] (BleuScorer's counts), "rouge" [C],
"cider" [C], "corpus" [6] (Bleu_1..4, ROUGE_L, CIDEr). The record flow: "ann" (annotation JSON
lines with non-ASCII characters and padded text), "records" (JSON, with a duplicate clip_id whose
later record wins) and "tvceval" (JSON, the reference's returned dict without METEOR). TVCEval runs
with its PTBTokenizer replaced by a whitespace tokenizer (the text is already tokenized) and METEOR
by a stub; both are Java.
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("HERO_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "caption_metrics_tiny.npz")
SEED = 5
WORDS = ["the", "a", "man", "woman", "is", "walks", "to", "door", "and", "says", "something",
         "house", "red", "car", "sits", "on", "chair", "looks", "at", "her", "phone", "while",
         "talking", "with", "friend", "n't", "'s", "kitchen", "opens", "window"]


def zipf_words(rng, n):
    p = 1.0 / np.arange(1, len(WORDS) + 1)
    return [WORDS[i] for i in rng.choice(len(WORDS), n, p=p / p.sum())]


def build_corpus(rng):
    hyps, refs = [], []

    def add(h, rs):
        hyps.append(" ".join(h))
        refs.append([" ".join(r) for r in rs])

    for _ in range(24):                                  # random clips; "the" in every clip
        rs = [["the"] + zipf_words(rng, rng.integers(7, 19))]
        rs += [zipf_words(rng, rng.integers(6, 18)) for _ in range(rng.integers(0, 4))]
        add(zipf_words(rng, rng.integers(5, 15)), rs)
    add([], [["the", "man", "walks"], ["a", "man", "walks", "to", "the", "door"]])   # empty hyp
    add(["the", "man"], [[], ["the", "woman", "sits"]])                              # empty ref
    add([], [[], ["the"]])                                                           # both empty
    add(["man"], [["man"], ["the", "door"]])                                         # one word
    add(["the"], [["the", "chair"], ["the"]])                                        # idf-0 only
    add(zipf_words(rng, 10), [["the"] + zipf_words(rng, 7), zipf_words(rng, 12)])    # tie 8 / 12
    add(["the", "man", "the", "man", "the", "man", "walks", "walks"],                # clipping
        [["the", "man", "walks"], ["the", "man", "the", "man"]])
    same = ["the", "woman", "opens", "the", "window", "and", "looks", "at", "her", "phone"]
    add(same, [list(same), ["a", "woman", "opens", "the", "door"]])                  # hyp == ref
    add(zipf_words(rng, 1024), [["the"] + zipf_words(rng, 40), zipf_words(rng, 1000)])
    return hyps, refs


def reference_scores(hyps, refs):
    sys.path.insert(0, os.path.join(REF, "eval"))
    from pycocoevalcap.bleu.bleu import Bleu
    from pycocoevalcap.bleu.bleu_scorer import BleuScorer
    from pycocoevalcap.cider.cider import Cider
    from pycocoevalcap.rouge.rouge import Rouge
    gts = {i: r for i, r in enumerate(refs)}
    res = {i: [h] for i, h in enumerate(hyps)}
    bleu, bleu_list = Bleu(4).compute_score(gts, res)
    scorer = BleuScorer(n=4)
    for i in gts:
        scorer += (res[i][0], gts[i])
    correct = np.array([c["correct"] for c in scorer.ctest], dtype=np.int64)
    reflen = np.array([min((abs(l - c["testlen"]), l) for l in c["reflen"])[1]
                       for c in scorer.ctest], dtype=np.int64)
    rouge, rouge_list = Rouge().compute_score(gts, res)
    cider, cider_list = Cider().compute_score(gts, res)
    return {"bleu": np.array(bleu_list, dtype=np.float64).T, "correct": correct, "reflen": reflen,
            "rouge": np.asarray(rouge_list, dtype=np.float64),
            "cider": np.asarray(cider_list, dtype=np.float64),
            "corpus": np.array(list(bleu) + [rouge, cider], dtype=np.float64)}


def reference_tvceval(ann_text, records):
    """eval/tvc.py:TVCEval as written, with the Java tokenizer and METEOR stubbed out."""
    sys.path.insert(0, REF)

    class WhitespaceTokenizer:
        def tokenize(self, captions_for_image):
            return {k: [" ".join(c.split()) for c in v] for k, v in captions_for_image.items()}

    class NoMeteor:
        def compute_score(self, gts, res):
            return 0.0, []

    for name, attr, obj in (("eval.pycocoevalcap.tokenizer.ptbtokenizer", "PTBTokenizer",
                             WhitespaceTokenizer),
                            ("eval.pycocoevalcap.meteor.meteor", "Meteor", NoMeteor)):
        mod = types.ModuleType(name)
        setattr(mod, attr, obj)
        sys.modules[name] = mod
    from eval.tvc import TVCEval
    with tempfile.NamedTemporaryFile("w", suffix=".jsonl", delete=False) as f:
        f.write(ann_text)
    try:
        out = TVCEval(f.name)(records)
    finally:
        os.remove(f.name)
    out.pop("METEOR")
    return out


def build_records(hyps, refs):
    """Annotation lines and result records over the first 8 clips of the corpus."""
    lines, records = [], []
    for i in range(8):
        descs = [{"desc": "  " + r + (" café" if j == 0 and i == 2 else "") + " "}
                 for j, r in enumerate(refs[i])]
        lines.append(json.dumps({"vid_name": f"v{i}", "clip_id": 100 + i, "descs": descs}))
        records.append({"vid_name": f"v{i}", "clip_id": 100 + i, "ts": [0.0, 1.0],
                        "descs": [{"desc": " " + hyps[i] + ("’s" if i == 3 else "")}]})
    # the first record of clip 105 is replaced by a later one
    records.insert(2, {"vid_name": "v5", "clip_id": 105, "ts": [0.0, 1.0],
                       "descs": [{"desc": "this caption is replaced"}]})
    return "\n".join(lines) + "\n", records


def main():
    rng = np.random.default_rng(SEED)
    hyps, refs = build_corpus(rng)
    one = (["the man walks to the door"], [["a man walks to the door", "the man walks"]])
    arrays = {"corpus": np.array(json.dumps({"hyps": hyps, "refs": refs})),
              "one_clip": np.array(json.dumps({"hyps": one[0], "refs": one[1]}))}
    for prefix, (h, r) in (("main.", (hyps, refs)), ("one.", one)):
        for k, v in reference_scores(h, r).items():
            arrays[prefix + k] = v
    ann, records = build_records(hyps, refs)
    arrays["ann"] = np.array(ann)
    arrays["records"] = np.array(json.dumps(records))
    arrays["tvceval"] = np.array(json.dumps(reference_tvceval(ann, records)))
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, {k: v.shape for k, v in arrays.items()})
    print(json.loads(str(arrays["tvceval"])))


if __name__ == "__main__":
    main()
