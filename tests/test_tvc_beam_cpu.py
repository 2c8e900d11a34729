"""TVC beam search (TvcGenerator.beam_search / beam_ids) with hero_b200.ops routed through
tests/fake_beam_ops.py, against the torch beam search over the reference's decoder
(tests/golden/tvc_beam_tiny.npz, written by tools/gen_tvc_beam_golden.py): the hypotheses kept at
every step, B = 1 against greedy decoding, the plan's beam arrays, the final pick, the bounds and
the evaluation records. The kernels are covered by test_tvc_beam_gpu.py."""
import json

import numpy as np
import pytest
import torch

from tests import fake_beam_ops
from tests import golden_util as gu
from tests import test_tvc_cpu as tvc


def golden():
    return gu.load("tvc_beam_tiny.npz")


def recording(monkeypatch):
    """Wraps ops.beam_select so that the token histories kept after every step are recorded:
    returns the list that receives one host [R, t + 1] tensor per step."""
    from hero_b200 import ops
    seen = []
    select = ops.beam_select

    def spy(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, *, beam, step, max_step,
            eos):
        select(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, beam=beam, step=step,
               max_step=max_step, eos=eos)
        R = logp.shape[0]
        seen.append(state_out[3].view(R, max_step)[:, :step + 1].cpu().clone())
    monkeypatch.setattr(ops, "beam_select", spy)
    return seen


def beam_agreement(seen, g, beam, thr):
    """Compare the hypotheses kept after every step with the golden's, as sets per caption (the
    order of the kept beams does not change the next step's candidates), up to each caption's
    first step whose selection margin is within `thr`: past it a rounding difference may keep
    another hypothesis. Returns the number of (caption, step) pairs compared."""
    steps, margin = g[f"b{beam}_steps"], g[f"b{beam}_margin"]
    n_cap, T = margin.shape
    assert len(seen) == T
    compared = 0
    for n in range(n_cap):
        low = np.flatnonzero(margin[n] <= thr)
        first = int(low[0]) if low.size else T
        for t in range(first):
            got = sorted(map(tuple, seen[t][n * beam:(n + 1) * beam].tolist()))
            want = sorted(map(tuple, steps[n, t, :, :t + 1].tolist()))
            assert got == want, (beam, n, t)
            compared += 1
    return compared


def logits_bound(tx):
    """The bound test_tvc_cpu puts on the teacher-forced logits: 2e-2 of the largest."""
    return 2e-2 * float(np.abs(tx["logits"]).max())


def generator(model, tx, eos=None):
    from hero_b200 import synth
    from hero_b200.tvc import TvcGenerator
    c = json.loads(str(tx["config"]))
    return TvcGenerator(model, c["max_step"], synth.BOS, synth.EOS if eos is None else eos, False)


@pytest.mark.parametrize("beam", [1, 3, 5])
def test_hypotheses_match_reference_beam_search(tmp_path, monkeypatch, beam):
    fake_beam_ops.install(monkeypatch)
    tx, g = tvc.fixture(), golden()
    model = tvc.tvc_model(tmp_path, tx)
    seen = recording(monkeypatch)
    gen = generator(model, tx)
    ids, score = gen.beam_ids(tvc.tvc_batch(tx, "val"), beam)
    thr = logits_bound(tx)
    compared = beam_agreement(seen, g, beam, thr)
    print(f"B = {beam}: {compared} (caption, step) pairs compared with the reference")
    assert compared > 0
    assert ids.shape == (g[f"b{beam}_margin"].shape[0], g["max_step"]) and ids.dtype == torch.int32
    assert score.dtype == torch.float32
    # captions whose every step is past the margin and whose pick is clear: the same caption
    clear = (g[f"b{beam}_margin"] > thr).all(1) & (g[f"b{beam}_a0_pick_gap"] > thr)
    for n in np.flatnonzero(clear):
        assert ids[n].tolist() == g[f"b{beam}_steps"][n, -1, g[f"b{beam}_a0_pick"][n]].tolist()


def test_beam_of_one_is_greedy(tmp_path, monkeypatch):
    fake_beam_ops.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    gen = generator(model, tx)
    want = gen.greedy_decode(tvc.tvc_batch(tx, "val"))
    assert gen.beam_search(tvc.tvc_batch(tx, "val"), 1) == want


def test_beam_arrays():
    from hero_b200.plan import ReprPlan, TvcPlan
    tx = tvc.fixture()
    b = tvc.tvc_batch(tx)
    p = TvcPlan(b["clip_ranges"], ReprPlan(b))
    T, B = 4, 3
    a = p.beam_arrays(T, B)
    R = p.n_seg * B
    assert a["beam_kv_off"].tolist() == [o for o in p.kv_off.tolist() for _ in range(B)]
    assert a["beam_kv_len"].tolist() == [n for n in p.kv_len.tolist() for _ in range(B)]
    assert a["beam_step_pos"].reshape(T, R)[2].tolist() == [2] * R
    assert a["beam_step_len"].reshape(T, R)[2].tolist() == [3] * R
    s0 = a["beam_state0"]
    assert s0.dtype == np.int32 and s0.size == R * T + 3 * R
    assert (s0[:R * T] == 0).all() and (s0[R * T + R:] == 0).all()
    score = s0[R * T:R * T + R].view(np.float32)
    assert score.tolist() == ([0.0] + [-np.inf] * (B - 1)) * p.n_seg
    anc = a["beam_anc0"].reshape(R, T)
    assert anc[:, 0].tolist() == list(range(R))
    for v in a.values():
        assert v.dtype == np.int32


def test_pick_honours_length_penalty_and_ties():
    from hero_b200.tvc import TvcGenerator
    score = np.array([[-4.0, -4.5, -9.0], [-2.0, -2.0, -3.0]], np.float32)
    length = np.array([[4, 6, 12], [3, 3, 5]], np.int32)
    assert TvcGenerator.pick_beam(score, length, 0.0).tolist() == [0, 0]     # tie: lower beam
    # -1, -0.75, -0.75 (tie: lower beam) and -0.67, -0.67, -0.6
    assert TvcGenerator.pick_beam(score, length, 1.0).tolist() == [1, 2]
    # -2, -1.84, -2.60 and -1.15, -1.15, -1.34
    assert TvcGenerator.pick_beam(score, length, 0.5).tolist() == [1, 0]


def test_finished_beams_emit_eos_and_the_pick_follows_the_scores(tmp_path, monkeypatch):
    """With EOS set to a token the search emits early, beams finish: after the first EOS a beam
    emits only EOS, its length stops, and beam_ids returns the beam with the best score / len **
    alpha, cut at EOS by beam_search."""
    from hero_b200 import ops
    fake_beam_ops.install(monkeypatch)
    tx, g = tvc.fixture(), golden()
    model = tvc.tvc_model(tmp_path, tx)
    eos = int(g["b3_steps"][0, 1, 0, 1])               # a token the B = 3 search emits at step 1
    finals = []
    select = ops.beam_select

    def spy(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, **kw):
        select(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, **kw)
        if kw["step"] == kw["max_step"] - 1:
            finals.append([x.cpu().clone() for x in state_out])
    monkeypatch.setattr(ops, "beam_select", spy)
    gen = generator(model, tx, eos=eos)
    for alpha in (0.0, 1.0):
        finals.clear()
        ids, score = gen.beam_ids(tvc.tvc_batch(tx, "val"), 3, alpha)
        s, fin, ln, hist = finals[0]
        T = ids.shape[1]
        hist = hist.view(-1, T)
        n_fin = 0
        for r in range(hist.shape[0]):
            row = hist[r].tolist()
            if eos in row:
                first = row.index(eos)
                assert row[first:] == [eos] * (T - first) and ln[r] == first + 1 and fin[r]
                n_fin += 1
            else:
                assert ln[r] == T and not fin[r]
        assert n_fin > 0
        best = gen.pick_beam(s.view(-1, 3).numpy(), ln.view(-1, 3).numpy(), alpha)
        rows = np.arange(len(best)) * 3 + best
        assert torch.equal(ids, hist[rows].int()) and torch.equal(score, s[rows])
        cut = gen.beam_search(tvc.tvc_batch(tx, "val"), 3, alpha)
        assert cut == [gen.cut_eos(r) for r in ids.tolist()]


def test_bounds_raise_before_any_op(tmp_path, monkeypatch):
    from hero_b200.tvc import TvcGenerator
    fake_beam_ops.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)

    def no_encode(batch):
        raise AssertionError("an op ran before the bounds were checked")
    monkeypatch.setattr(model, "encode", no_encode)
    b = tvc.tvc_batch(tx, "val")
    for bad in (0, 17, -1):
        with pytest.raises(ValueError, match="beam_size"):
            generator(model, tx).beam_ids(b, bad)
    for bad in (0, 1024):
        with pytest.raises(ValueError, match="max_step"):
            TvcGenerator(model, bad, 0, 2, False).beam_search(b, 3)
    for bad in (-0.5, float("nan")):
        with pytest.raises(ValueError, match="length_penalty"):
            generator(model, tx).beam_search(b, 3, bad)
    fe = model.v_encoder.f_encoder
    monkeypatch.setattr(fe, "vocab_pad", fe.embeddings.word_embeddings.weight.shape[0] - 4)
    with pytest.raises(ValueError, match="beam_size"):
        generator(model, tx).beam_ids(b, 5)          # more beams than vocabulary entries


def test_kernel_wrappers_check_bounds_before_launch():
    from hero_b200 import ops
    x = torch.zeros(2, 8)
    lse, lp, ci = torch.zeros(2), torch.zeros(2, 16), torch.zeros(2, 16, dtype=torch.int32)
    for beam, n in ((0, 8), (17, 8), (4, 3), (2, 9)):
        with pytest.raises(ValueError, match="beam_logprob_topk"):
            ops.beam_logprob_topk(x, n, beam, lse, lp, ci)
    st = (torch.zeros(6), torch.zeros(6, dtype=torch.int32), torch.zeros(6, dtype=torch.int32),
          torch.zeros(12, dtype=torch.int32))
    a = torch.zeros(12, dtype=torch.int32)
    for beam, step in ((4, 0), (3, 2), (3, -1)):
        with pytest.raises(ValueError, match="beam_select"):
            ops.beam_select(torch.zeros(6, beam), torch.zeros(6, beam, dtype=torch.int32), st, a,
                            st, a, st[1], beam=beam, step=step, max_step=2, eos=2)
    z = torch.zeros(2, 128, dtype=torch.bfloat16)
    idx = torch.zeros(2, 4, dtype=torch.int32)
    for kw in (dict(max_kv_len=1025), dict(max_kv_len=5), dict(max_kv_len=4, head_dim=32)):
        with pytest.raises(ValueError, match="dec_attn_gather_fwd"):
            ops.dec_attn_gather_fwd(z, z, z, idx, idx[:, 0], z, heads=2, **kw)


def test_decode_tvc_beam_records(tmp_path, monkeypatch):
    from hero_b200 import evalpass, synth
    fake_beam_ops.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    c = json.loads(str(tx["config"]))
    vb = synth.syn_tvc_batch(**c["batch_args"], split="val")
    loader = [vb, dict(vb)]
    kw = dict(max_step=c["max_step"], bos=synth.BOS, eos=synth.EOS, tokenizer=tvc._Stub())
    greedy = evalpass.decode_tvc(model, loader, **kw)
    assert evalpass.decode_tvc(model, loader, beam_size=1, **kw) == greedy
    recs = evalpass.decode_tvc(model, loader, beam_size=3, length_penalty=1.0, **kw)
    want = generator(model, tx).beam_search(vb, 3, 1.0)
    assert len(recs) == 2 * len(vb["clip_ids"])
    for r, g, ids in zip(recs, greedy, want * 2):
        assert set(r) == {"vid_name", "clip_id", "ts", "descs"}
        assert (r["vid_name"], r["clip_id"], r["ts"]) == (g["vid_name"], g["clip_id"], g["ts"])
        assert r["descs"] == [{"desc": " ".join(f"w{i}" for i in ids)}]
    with pytest.raises(ValueError, match="length_penalty"):
        evalpass.decode_tvc(model, loader, beam_size=3, length_penalty=-1.0, **kw)
