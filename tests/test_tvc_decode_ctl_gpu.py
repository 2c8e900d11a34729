"""TVC decoding controls on the H100: hero_dec_ban_tokens against its restatement bit for bit
(both history layouts, a real beam-state slab, n up to 8, steps up to 1023, vocabulary 50 272),
hero_sample_tokens against rank_topk(k=1) (rows without an exact tie at the maximum, where
top_k=1 draws among the tied columns) and its restatement, the column with a row's largest uniform
never overriding a banned or a far lower logit, the sampled distribution against the
renormalised target (chi-square) and the kept set, and at real dimensions greedy and B = 5 beam
hypotheses against the same rules over the reference decoder staged under oracle/_ref, the caption
properties, and every decode loop without host synchronisation."""
import math

import numpy as np
import pytest
import torch

from tests import fake_decode_ctl_ops as fdc
from tests import test_tvc_beam_cpu as beam_cpu
from tests import test_tvc_beam_gpu as beam_gpu
from tests import test_tvc_decode_ctl_cpu as ctl_cpu
from tests import test_tvc_gpu as tvc_gpu
from tests import test_videoqa_gpu as qa_gpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
V_REAL = 50272


def _histories(rows, T, gen, alphabet):
    """Token histories [rows, T] over a small alphabet spread across the vocabulary, with copied
    stretches, so n-grams of every size recur."""
    pool = torch.tensor([3, 17, 999, 25000, V_REAL - 8, 40000, 7, 12345][:alphabet])
    h = pool[torch.randint(0, alphabet, (rows, T), generator=gen)]
    for r in range(rows):
        a = int(torch.randint(0, T // 2, (1,), generator=gen))
        k = int(torch.randint(2, 40, (1,), generator=gen))
        b = a + k + int(torch.randint(0, 5, (1,), generator=gen))
        k = max(0, min(k, T - b))
        h[r, b:b + k] = h[r, a:a + k].clone()
    h[0, 5] = V_REAL + 3                      # a token outside the columns: never written
    return h.int()


@pytest.mark.parametrize("layout", ["greedy", "beam"])
def test_ban_tokens_matches_restatement(layout):
    from hero_b200 import ops
    from hero_b200.tvc import _beam_state
    gen = torch.Generator().manual_seed(11)
    rows, T, n_valid, bos, eos = 6, 1024, V_REAL - 7, 0, 2
    steps = (0, 1, 2, 3, 7, 8, 64, 511, 1000, 1023)
    n_banned = 0
    for n in range(1, 9):
        h = _histories(rows, T, gen, 2 + n % 5)
        if layout == "greedy":               # out [T + 1, rows], history out[1:]
            out = torch.cat([torch.full((1, rows), bos, dtype=torch.int32), h.t()], 0).to(DEV)
            hist, ss, rs = out[1:], rows, 1
        else:                                # the history slab of a real beam state
            slab = torch.zeros(rows * T + 3 * rows, dtype=torch.int32, device=DEV)
            hist = _beam_state(slab, rows, T)[3]
            hist.copy_(h.reshape(-1).to(DEV))
            ss, rs = 1, T
        for t in steps:
            for min_len in (0, 5):
                x = torch.randn(rows, V_REAL + 16, generator=gen).to(DEV)
                want = x.clone()
                ops.ban_tokens(x, n_valid, hist, step_stride=ss, row_stride=rs, bos=bos, step=t,
                               ngram=n, min_length=min_len, eos=eos)
                fdc.ban_tokens(want, n_valid, hist, step_stride=ss, row_stride=rs, bos=bos,
                               step=t, ngram=n, min_length=min_len, eos=eos)
                assert torch.equal(x, want), (layout, n, t, min_len)
                n_banned += int(torch.isinf(x).sum())
    assert n_banned > 100


def _logits(rows, V, gen, ld_pad=24, scale=3.0):
    x = (scale * torch.randn(rows, V + ld_pad, generator=gen)).to(DEV)
    return x


def test_top_k_1_is_rank_topk():
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(2)
    for V in (120, V_REAL):
        x = _logits(37, V, gen)
        x[3, V - 1] = 80.0
        x[4, 10] = float("-inf")
        val = torch.empty(37, 1, device=DEV)
        want = torch.empty(37, 1, dtype=torch.int32, device=DEV)
        ops.rank_topk(x, V, 1, val, want)
        for kw in (dict(), dict(temperature=0.7), dict(top_p=0.5), dict(temperature=2.0, top_p=0.9)):
            ids = torch.full((37,), -1, dtype=torch.int32, device=DEV)
            ops.sample_tokens(x, V, ids, top_k=1, seed=5, step=3, **dict(
                dict(temperature=1.0, top_p=1.0), **kw))
            assert torch.equal(ids, want[:, 0]), (V, kw)


def test_largest_uniform_cannot_override_the_logits():
    """The kernel on the row whose column gets the largest uniform (found by the restatement's
    hash): banned (-inf) or 40 below the others that column is never drawn, 40 above them it is;
    every row agrees with the restatement where its draw is clear."""
    from hero_b200 import ops
    row, col = ctl_cpu.largest_uniform_row()
    n = V_REAL
    x = torch.randn(row + 1, n, generator=torch.Generator().manual_seed(0)).to(DEV)
    ids = torch.empty(row + 1, dtype=torch.int32, device=DEV)
    for kw in (dict(top_k=0, top_p=1.0), dict(top_k=0, top_p=0.999), dict(top_k=n - 1, top_p=1.0)):
        for val, drawn in ((-math.inf, False), (-40.0, False), (40.0, True)):
            x[row, col] = val
            ops.sample_tokens(x, n, ids, temperature=1.0, seed=123, step=4, **kw)
            assert (int(ids[row]) == col) == drawn, (kw, val)
            want, v = fdc.sample_ref(x, n, temperature=1.0, seed=123, step=4, **kw)
            top = v.topk(2, dim=1).values
            clear = (top[:, 0] - top[:, 1]) > 1e-4
            assert torch.equal(ids.long()[clear], want[clear]), (kw, val)


SETTINGS = [dict(), dict(temperature=0.7), dict(top_k=20), dict(top_p=0.9),
            dict(top_k=20, top_p=0.9)]


def test_sample_matches_restatement_where_the_draw_is_clear():
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(4)
    for V in (300, V_REAL):
        x = _logits(64, V, gen)
        for i, kw in enumerate(SETTINGS):
            kw = dict(dict(temperature=1.0, top_k=0, top_p=1.0), **kw)
            ids = torch.empty(64, dtype=torch.int32, device=DEV)
            ops.sample_tokens(x, V, ids, seed=1000 + i, step=7, **kw)
            want, v = fdc.sample_ref(x, V, seed=1000 + i, step=7, **kw)
            top = v.topk(2, dim=1).values
            clear = (top[:, 0] - top[:, 1]) > 1e-4
            assert int(clear.sum()) >= 48
            assert torch.equal(ids.long()[clear], want[clear]), (V, kw)
            # bit-for-bit repeatable
            again = torch.empty_like(ids)
            ops.sample_tokens(x, V, again, seed=1000 + i, step=7, **kw)
            assert torch.equal(again, ids)


def _target(z, temperature, top_k, top_p):
    """fp64 renormalised target over one row and the nominal top_p moved to the middle between
    two cumulative masses (so fp32 and fp64 agree on the kept set)."""
    x = z.double() / temperature
    order = torch.argsort(x, descending=True)
    keep = torch.zeros_like(x, dtype=torch.bool)
    n = len(x) if top_k == 0 else top_k
    keep[order[:n]] = True
    p = torch.softmax(torch.where(keep, x, torch.full_like(x, -math.inf)), 0)
    if top_p < 1.0:
        cum = torch.cumsum(p[order], 0)
        m = int(torch.nonzero(cum >= top_p)[0])
        top_p = float((cum[m - 1] + cum[m]) / 2) if m > 0 else float(cum[0] / 2)
        m = int(torch.nonzero(cum >= top_p)[0])
        keep = torch.zeros_like(keep)
        keep[order[:m + 1]] = True
        p = torch.softmax(torch.where(keep, x, torch.full_like(x, -math.inf)), 0)
    return p, keep, top_p


def test_sampled_distribution_chi_square():
    from scipy.stats import chisquare
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(8)
    V, rows = 300, 65536
    z = 2.0 * torch.randn(V, generator=gen)
    x = z.to(DEV).expand(rows, V).contiguous()
    for i, kw in enumerate(SETTINGS):
        kw = dict(dict(temperature=1.0, top_k=0, top_p=1.0), **kw)
        p, keep, top_p = _target(z, kw["temperature"], kw["top_k"], kw["top_p"])
        kw["top_p"] = top_p
        ids = torch.empty(rows, dtype=torch.int32, device=DEV)
        ops.sample_tokens(x, V, ids, seed=31 + i, step=2, **kw)
        counts = torch.bincount(ids.long().cpu(), minlength=V).double()
        assert counts[~keep].sum() == 0, kw                    # nothing outside the kept set
        exp = p[keep] * rows
        obs = counts[keep]
        big = exp >= 5
        o = torch.cat([obs[big], obs[~big].sum().view(1)]) if (~big).any() else obs[big]
        e = torch.cat([exp[big], exp[~big].sum().view(1)]) if (~big).any() else exp[big]
        pv = chisquare(o.numpy(), e.numpy()).pvalue
        print(f"{kw}: {int(keep.sum())} kept, chi-square p = {pv:.3g}")
        assert pv > 1e-3, kw


def test_draws_stay_in_the_kept_set():
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(6)
    rows = 256
    x = _logits(rows, V_REAL, gen, scale=4.0)
    for i, kw in enumerate([dict(top_k=50), dict(top_p=0.9), dict(top_k=300, top_p=0.8),
                            dict(temperature=0.5, top_p=0.95)]):
        kw = dict(dict(temperature=1.0, top_k=0, top_p=1.0), **kw)
        ids = torch.empty(rows, dtype=torch.int32, device=DEV)
        ops.sample_tokens(x, V_REAL, ids, seed=77 + i, step=1, **kw)
        xs = x[:, :V_REAL] / torch.tensor(kw["temperature"], dtype=torch.float32)
        keep = fdc.kept_mask(xs, kw["top_k"], kw["top_p"])
        assert keep.gather(1, ids.long()[:, None]).all(), kw
        assert int(keep.sum(1).max()) < V_REAL


# ------------------------------------------------------------------ real dimensions
def _masked(last_logits, n, min_len, eos, n_valid):
    """The same rules restated over the reference's last-position logits: inputs are [bos] + the
    history, so the n-gram bans come straight from them."""
    def last(inputs):
        z = last_logits(inputs).clone()
        t = inputs.shape[1] - 1
        for r in range(inputs.shape[0]):
            for c in ctl_cpu.brute_force_bans(inputs[r].tolist(), n):
                if c < n_valid:
                    z[r, c] = -math.inf
        if t < min_len:
            z[:, eos] = -math.inf
        return z
    return last


def test_real_dimensions_against_reference_with_controls(monkeypatch):
    import tools.gen_tvc_beam_golden as gb
    from hero_b200 import ops, synth
    from hero_b200.tvc import TvcGenerator
    VideoModelConfig, _ = qa_gpu._reference_module()
    from model.tvc import HeroForTvc as RefTvc
    model, path = beam_gpu._real()
    T, eos, bos, n, min_len, B = 20, synth.EOS, synth.BOS, 3, 5, 5
    hb = synth.syn_tvc_batch(n_videos=4, seed=9, vocab=50265, split="val")
    db = lambda: synth.to_device(hb, DEV)   # noqa: E731
    gen = TvcGenerator(model, T, bos, eos, fp16=False, min_length=min_len,
                       no_repeat_ngram_size=n)
    greedy = gen.decode_ids(db())
    ids, score = gen.beam_ids(db(), B)
    sampled = gen.sample_ids(db(), top_p=0.9, seed=3)
    for rows in (greedy, ids, sampled):
        ctl_cpu.check_properties(rows.tolist(), n, min_len, eos, bos)
    fe = model.v_encoder.f_encoder
    n_valid = fe.embeddings.word_embeddings.weight.shape[0] - fe.vocab_pad
    ref = RefTvc(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(model.state_dict())
    ref = ref.to(DEV).eval()
    N = ids.shape[0]
    with torch.no_grad():
        want1 = gb.beam_search(_masked(gb.reference_last_logits(ref, db(), 1), n, min_len, eos,
                                       n_valid), N, 1, T, bos, eos, n_valid)
        want = gb.beam_search(_masked(gb.reference_last_logits(ref, db(), B), n, min_len, eos,
                                      n_valid), N, B, T, bos, eos, n_valid)
        lp = beam_gpu._forced_logprobs(model, db(), ids, bos, n_valid)
        inp = torch.cat([torch.full((N, 1), bos, dtype=torch.long), ids[:, :-1].long()],
                        1).to(DEV)
        zr = ref.decode(ref.encode(db()), db()["cap_attn_mask"], inp,
                        torch.arange(T).unsqueeze(0).to(DEV), None,
                        compute_loss=False)[..., :n_valid].float()
        lr = torch.log_softmax(zr, dim=-1)
    thr = 2 * float((lp - lr).abs().max())
    # greedy: up to each caption's first EOS and its first step with a margin within thr
    compared1 = 0
    for r in range(N):
        row = greedy[r].tolist()
        stop = row.index(eos) + 1 if eos in row else T
        low = np.flatnonzero(want1["margin"][r] <= thr)
        stop = min(stop, int(low[0]) if low.size else T)
        if stop:
            assert row[:stop] == want1["steps"][r, stop - 1, 0, :stop].tolist(), r
        compared1 += stop
    # beam: the hypotheses kept after every step
    seen = []
    select = ops.beam_select

    def spy(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, **kw):
        select(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, **kw)
        seen.append(state_out[3].view(-1, T)[:, :kw["step"] + 1].cpu().clone())
    monkeypatch.setattr(ops, "beam_select", spy)
    gen.beam_ids(db(), B)
    compared = beam_cpu.beam_agreement(seen, {f"b{B}_steps": want["steps"],
                                              f"b{B}_margin": want["margin"]}, B, thr)
    print(f"real dimensions, n = {n}, min_length = {min_len}: margin {thr:.4f}, greedy "
          f"{compared1} positions and B = {B} {compared} (caption, step) pairs compared")
    assert compared1 > 0 and compared > 0


def test_decode_loops_with_controls_make_one_copy_and_no_sync():
    from torch.profiler import ProfilerActivity, profile
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    from hero_b200.tvc import TvcGenerator
    model, _ = tvc_gpu._tvc_model(layers=(2, 2, 2), hidden=256, heads=4, vocab=1000)
    model = model.to(DEV).eval()
    b = attach_plan(synth.syn_tvc_batch(n_videos=8, seed=4, vfeat_dim=64, vocab=1000,
                                        split="val"))
    gen = TvcGenerator(model, 30, synth.BOS, synth.EOS, fp16=False, min_length=4,
                       no_repeat_ngram_size=2)
    calls = {"greedy": lambda d: gen.greedy_decode(d), "beam": lambda d: gen.beam_search(d, 4),
             "sample": lambda d: gen.sample(d, temperature=0.9, top_k=50, top_p=0.9, seed=7)}
    for name, call in calls.items():
        first = call(synth.to_device(b, DEV))                 # warm-up
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = call(synth.to_device(b, DEV))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert out == first and len(out) == len(b["clip_ids"]), name
        ctl_cpu.check_properties([r + [synth.EOS] for r in out], 2, 4, synth.EOS, synth.BOS)
        db = synth.to_device(b, DEV)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(db)
            torch.cuda.synchronize()
        d2h = [e for e in prof.events() if "Memcpy DtoH" in e.name]
        assert len(d2h) == 1, (name, [e.name for e in d2h])
