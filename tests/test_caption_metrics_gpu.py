"""TVC caption metrics on the kernels of csrc/capeval.cu: the reference's scores
(tests/golden/caption_metrics_tiny.npz) with BLEU and ROUGE-L bit for bit and CIDEr-D within 1e-12
relative, the same agreement with the plain restatement (tests/fake_caption_ops.py) on seeded
corpora of about 11 000 clips, bitwise repeatability, and a device pass that never synchronises and
ends in one device-to-host copy."""
import json

import numpy as np
import pytest
import torch

from hero_b200 import capeval, synth
from tests import fake_caption_ops
from tests import golden_util as gu
from tests.test_caption_metrics_cpu import _corpus, check_against_golden, check_tvceval_flow

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prefix, key", [("main.", "corpus"), ("one.", "one_clip")])
def test_golden_parity(prefix, key):
    fx = gu.load("caption_metrics_tiny.npz")
    scores, per_clip = capeval.caption_scores(*_corpus(fx, key))
    check_against_golden(fx, prefix, scores, per_clip)


def test_tvceval_record_flow(tmp_path):
    check_tvceval_flow(gu.load("caption_metrics_tiny.npz"), tmp_path)


@pytest.mark.parametrize("seed", [0, 1])
def test_random_corpus_against_restatement(seed):
    hyps, refs = synth.syn_captions(11000, seed=seed, n_refs=(1, 5), ref_len=(0, 24),
                                    hyp_len=(0, 20), vocab=20000, n_long=6)
    pack = capeval.CaptionPack(hyps, refs)
    got = capeval.device_stats(pack).cpu().numpy()
    want = fake_caption_ops.caption_stats(*[torch.from_numpy(np.ascontiguousarray(a, np.int32))
                                            for a in (pack.sent_off, pack.gram_off, pack.ref_off,
                                                      pack.tok)],
                                          torch.from_numpy(pack.log_n), n_grams=pack.n_grams,
                                          n_ref_grams=pack.n_ref_grams,
                                          max_hyp_grams=pack.max_hyp_grams).numpy()
    C = pack.n_clips
    ints = np.r_[np.arange(5 * C), 5 * C + 4 + 5 * np.arange(len(got) // 5 - C)]
    assert np.array_equal(got[ints], want[ints])                 # BLEU counts, lengths, LCS
    sim = np.setdiff1d(np.arange(len(got)), ints)
    np.testing.assert_allclose(got[sim], want[sim], rtol=1e-12, atol=1e-300)
    s_got, c_got = capeval.finish(pack, got)
    s_want, c_want = capeval.finish(pack, want)
    for k in capeval.METRICS[:5]:
        assert s_got[k] == s_want[k], k
    assert np.array_equal(c_got["bleu"], c_want["bleu"])
    assert np.array_equal(c_got["rouge_l"], c_want["rouge_l"])
    np.testing.assert_allclose(c_got["cider"], c_want["cider"], rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(s_got["CIDEr"], s_want["CIDEr"], rtol=1e-12, atol=0)


def test_two_runs_are_bitwise_equal():
    hyps, refs = synth.syn_captions(3000, seed=7, n_long=4)
    pack = capeval.CaptionPack(hyps, refs)
    a = capeval.device_stats(pack).cpu().numpy()
    b = capeval.device_stats(pack).cpu().numpy()
    assert a.tobytes() == b.tobytes()


def test_device_pass_does_not_synchronise(monkeypatch):
    hyps, refs = synth.syn_captions(2000, seed=3)
    pack = capeval.CaptionPack(hyps, refs)
    capeval.device_stats(pack)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = capeval.device_stats(pack)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    copies = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(t, *a, **k):
        copies.append(tuple(t.shape))
        return real_cpu(t, *a, **k)

    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    scores, _ = capeval.caption_scores(hyps, refs)
    assert copies == [tuple(out.shape)]
    monkeypatch.undo()
    assert json.dumps(scores)        # plain floats
