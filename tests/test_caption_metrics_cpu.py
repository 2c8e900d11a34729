"""TVC caption metrics (hero_b200.capeval) on the CPU, with the device pass replaced by its plain
restatement (tests/fake_caption_ops.py): host packing and the vocabulary, the bounds, the key-set
check of TVCEval, the tokenizer rules, and parity with the reference's COCO scorers
(tests/golden/caption_metrics_tiny.npz, tools/gen_caption_metrics_golden.py). The kernels
themselves are covered by tests/test_caption_metrics_gpu.py."""
import json

import numpy as np
import pytest

from hero_b200 import capeval, ops
from tests import fake_caption_ops
from tests import golden_util as gu


def _corpus(fx, key):
    c = json.loads(str(fx[key]))
    return [h.split() for h in c["hyps"]], [[r.split() for r in rs] for rs in c["refs"]]


def check_against_golden(fx, prefix, scores, per_clip):
    """BLEU and ROUGE-L bit for bit, CIDEr-D within 1e-12 relative, per clip and for the corpus."""
    want = fx[prefix + "corpus"]
    got = np.array([scores[k] for k in capeval.METRICS])
    assert np.array_equal(got[:5], want[:5]), (got, want)
    np.testing.assert_allclose(got[5], want[5], rtol=1e-12, atol=0)
    assert np.array_equal(per_clip["correct"], fx[prefix + "correct"])
    assert np.array_equal(per_clip["reflen"], fx[prefix + "reflen"])
    assert np.array_equal(per_clip["bleu"], fx[prefix + "bleu"])
    assert np.array_equal(per_clip["rouge_l"], fx[prefix + "rouge"])
    np.testing.assert_allclose(per_clip["cider"], fx[prefix + "cider"], rtol=1e-12, atol=1e-300)


def test_pack_vocabulary_and_offsets():
    hyps = [["a", "b", "a"], []]
    refs = [[["b", "c"]], [["a"], ["c", "c", "d", "e", "f"]]]
    p = capeval.CaptionPack(hyps, refs)
    assert p.vocab_size == 6
    assert p.tok.tolist() == [1, 2, 1, 2, 3, 1, 3, 3, 4, 5, 6]     # ids by first appearance
    assert p.sent_off.tolist() == [0, 3, 3, 5, 6, 11]
    assert p.lens.tolist() == [3, 0, 2, 1, 5]
    # n-grams per sentence: sum over n = 1..4 of max(0, len - n + 1)
    assert p.gram_off.tolist() == [0, 6, 6, 9, 10, 24]
    assert p.ref_off.tolist() == [0, 1, 3]
    assert (p.n_grams, p.n_ref_grams, p.max_hyp_grams) == (24, 18, 6)
    assert p.log_n[1:].tolist() == [np.log(1.0), np.log(2.0)]
    views = p.upload(capeval._device())
    assert [v.tolist() for v in views[:4]] == [p.sent_off.tolist(), p.gram_off.tolist(),
                                              p.ref_off.tolist(), p.tok.tolist()]
    assert views[4].tolist() == p.log_n.tolist()


def _no_launch(*a, **k):
    raise AssertionError("ops.caption_stats must not run")


@pytest.mark.parametrize("case", ["long_hyp", "long_ref", "vocab", "no_ref", "count", "empty"])
def test_bounds_raise_before_launch(monkeypatch, case):
    monkeypatch.setattr(ops, "caption_stats", _no_launch)
    hyps, refs = [["a"], ["b"]], [[["a"]], [["b"], ["c"]]]
    if case == "long_hyp":
        hyps[1] = ["x"] * 1025
    elif case == "long_ref":
        refs[1][1] = ["x"] * 1025
    elif case == "vocab":
        hyps[0] = [str(i) for i in range(65536)][:1024]
        refs[0] = [[str(i) for i in range(j, j + 1024)] for j in range(1024, 65536, 1024)]
    elif case == "no_ref":
        refs[1] = []
    elif case == "count":
        refs = refs[:1]
    else:
        hyps, refs = [], []
    with pytest.raises(ValueError, match="caption_scores"):
        capeval.caption_scores(hyps, refs)


def test_bounds_accept_the_limits(monkeypatch):
    fake_caption_ops.install(monkeypatch)
    words = [str(i) for i in range(65535)]
    refs = [[words[j:j + 1024] for j in range(0, 65535, 1024)]]
    capeval.caption_scores([["0"] * 1024], refs)


def _write_ann(tmp_path, rows):
    path = tmp_path / "ann.jsonl"
    path.write_text("".join(json.dumps(r) + "\n" for r in rows))
    return str(path)


def test_tvceval_key_set_mismatch(tmp_path, monkeypatch):
    fake_caption_ops.install(monkeypatch)
    ann = _write_ann(tmp_path, [{"clip_id": i, "descs": [{"desc": "a man walks"}]}
                                for i in (1, 2, 3)])
    ev = capeval.TVCEval(ann, tokenize=None)
    rec = [{"clip_id": i, "descs": [{"desc": "a man"}]} for i in (1, 3, 7)]
    with pytest.raises(ValueError, match=r"missing \[2\], extra \[7\]"):
        ev(rec)
    out = ev(rec[:2] + [{"clip_id": 2, "descs": [{"desc": "a man"}]}])
    assert set(out) == set(capeval.METRICS)


@pytest.mark.parametrize("text, want", [
    ("A Man Walks", "a man walks"),                                      # lower-casing
    ("He stops. She waits, then leaves; done: yes? no! wait...", "he stops she waits then leaves "
     "done yes no wait"),                                                # . , ; : ? ! ...
    ('She says "hello" and \'bye\'', "she says hello and bye"),          # quotes
    ("It's his", "it 's his"),
    ("they're here", "they 're here"),
    ("we've gone", "we 've gone"),
    ("you'll see", "you 'll see"),
    ("he'd go", "he 'd go"),
    ("i'm here", "i 'm here"),
    ("don't", "do n't"),
    ("can't", "ca n't"),
    ("cannot", "can not"),
    ("gonna gotta wanna", "gon na got ta wan na"),
    ("a t-shirt - and -- more", "a t-shirt and more"),                   # hyphenated words
    ("3.5 pounds for 1,000 people.", "3.5 pounds for 1,000 people"),     # numbers
    ("Mr. Smith meets Dr. Jones etc.", "mr. smith meets dr. jones etc."),  # abbreviations
    ("in the U.S. today", "in the u.s. today"),                          # acronyms
    ("(smiles) [laughs] {x}", "smiles laughs x"),                        # brackets
    ("", ""),
])
def test_ptb_tokenize(text, want):
    assert capeval.ptb_tokenize(text) == want


@pytest.mark.parametrize("prefix, key", [("main.", "corpus"), ("one.", "one_clip")])
def test_golden_parity_through_fake_ops(monkeypatch, prefix, key):
    fake_caption_ops.install(monkeypatch)
    fx = gu.load("caption_metrics_tiny.npz")
    scores, per_clip = capeval.caption_scores(*_corpus(fx, key))
    check_against_golden(fx, prefix, scores, per_clip)


def check_tvceval_flow(fx, tmp_path):
    ann = tmp_path / "ann.jsonl"
    ann.write_text(str(fx["ann"]))
    got = capeval.TVCEval(str(ann), tokenize=None)(json.loads(str(fx["records"])))
    want = json.loads(str(fx["tvceval"]))
    assert list(got) == list(capeval.METRICS) and set(want) == set(got)
    for k in capeval.METRICS[:5]:
        assert got[k] == want[k], k
    np.testing.assert_allclose(got["CIDEr"], want["CIDEr"], rtol=1e-12, atol=0)


def test_tvceval_record_flow_through_fake_ops(monkeypatch, tmp_path):
    fake_caption_ops.install(monkeypatch)
    check_tvceval_flow(gu.load("caption_metrics_tiny.npz"), tmp_path)


def test_fake_lcs_matches_the_recurrence():
    rng = np.random.default_rng(0)
    for _ in range(200):
        a = tuple(rng.integers(1, 4, rng.integers(0, 12)).tolist())
        b = tuple(rng.integers(1, 4, rng.integers(0, 12)).tolist())
        L = np.zeros((len(a) + 1, len(b) + 1), dtype=int)
        for i in range(1, len(a) + 1):
            for j in range(1, len(b) + 1):
                L[i, j] = L[i - 1, j - 1] + 1 if a[i - 1] == b[j - 1] else max(L[i - 1, j],
                                                                             L[i, j - 1])
        assert fake_caption_ops._lcs(a, b) == L[-1, -1]
