"""TVC beam search on the H100: hero_beam_logprob_topk against fp64 torch, hero_dec_attn_gather_fwd
against the torch restatement and the range kernel, hero_beam_select against its restatement over
several ping-pong steps, the tiny fixture against the reference's beam search
(tests/golden/tvc_beam_tiny.npz) and, at real dimensions, B = 1 against greedy decoding, B = 5
against the same beam search over the reference staged under oracle/_ref, the returned scores
against the teacher-forced log-probabilities, and beam search without host synchronisation."""
import pytest
import torch

from tests import fake_beam_ops
from tests import test_tvc_beam_cpu as beam_cpu
from tests import test_tvc_cpu as cpu
from tests import test_tvc_gpu as tvc_gpu
from tests import test_videoqa_gpu as qa_gpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
BF16 = torch.bfloat16


@pytest.mark.parametrize("V", [120, 50272])
@pytest.mark.parametrize("beam", [1, 4, 16])
def test_logprob_topk_matches_fp64(V, beam):
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(V + beam)
    rows, ld = 37, V + 24                                  # a row stride larger than V
    x = (3 * torch.randn(rows, ld, generator=gen)).to(DEV)
    x[0, 5] = x[0, V - 2] = x[0, 17] = 40.0                # planted ties: lower columns first
    x[1, :] = 1.5                                          # a constant row: columns 0, 1, ...
    x[2, V:] = 1e9                                         # beyond n: not a candidate
    x[3, V - 1] = 50.0                                     # the last real column
    x[4, 7] = float("-inf")
    for xs in (x, x[:, 1:]):                               # 16-byte aligned rows, then unaligned
        lse = torch.empty(rows, device=DEV)
        logp = torch.empty(rows, beam, device=DEV)
        cols = torch.empty(rows, beam, dtype=torch.int32, device=DEV)
        n = V if xs is x else V - 1
        ops.beam_logprob_topk(xs, n, beam, lse, logp, cols)
        z = xs[:, :n].double()
        want_lse = torch.logsumexp(z, dim=1)
        order = torch.sort(xs[:, :n], dim=1, descending=True, stable=True).indices[:, :beam]
        assert torch.equal(cols.long(), order)
        torch.testing.assert_close(lse.double(), want_lse, rtol=1e-6, atol=1e-5)
        torch.testing.assert_close(logp.double(), z.gather(1, order) - want_lse[:, None],
                                   rtol=1e-6, atol=2e-5)
        if beam == 1:                                      # the greedy argmax, bit for bit
            idx = torch.empty(rows, 1, dtype=torch.int32, device=DEV)
            val = torch.empty(rows, 1, device=DEV)
            ops.rank_topk(xs, n, 1, val, idx)
            assert torch.equal(cols, idx)
            assert torch.equal(logp, val - lse[:, None])
        assert cols[1].tolist() == list(range(beam))
        assert cols[0, 0] == (5 if xs is x else 4)           # the planted column, shifted by one


def test_gather_attention_matches_torch_and_the_range_kernel():
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(5)
    heads, rows, T, n_kv = 12, 45, 30, 45 * 30
    H = heads * 64
    cache = torch.randn(n_kv, 3 * H, generator=gen).to(BF16).to(DEV)
    q, k, v = cache[:rows, :H], cache[:, H:2 * H], cache[:, 2 * H:]
    lens = torch.randint(1, T + 1, (rows,), generator=gen)
    lens[0], lens[1] = 1, T
    idx = torch.randint(0, n_kv, (rows, T), generator=gen).int()
    idx_d, len_d = idx.to(DEV), lens.int().to(DEV)
    out = torch.full((rows, H), float("nan"), dtype=BF16, device=DEV)
    ops.dec_attn_gather_fwd(q, k, v, idx_d, len_d, out, heads=heads, max_kv_len=T)
    ref = fake_beam_ops.dec_attn_gather_ref(q, k, v, idx_d, len_d, heads)
    assert not torch.isnan(out).any()
    torch.testing.assert_close(out.float(), ref, rtol=8e-3, atol=2e-3)
    assert torch.equal(out[0], v[int(idx[0, 0])])          # a single key returns its value row
    # contiguous ranges: bit for bit the range kernel
    off = torch.arange(rows, dtype=torch.int32) * T
    rng = (off[:, None] + torch.arange(T, dtype=torch.int32)[None, :]).to(DEV)
    a = torch.empty(rows, H, dtype=BF16, device=DEV)
    b = torch.empty(rows, H, dtype=BF16, device=DEV)
    ops.dec_attn_gather_fwd(q, k, v, rng, len_d, a, heads=heads, max_kv_len=T)
    ops.dec_attn_fwd(q, k, v, off.to(DEV), len_d, b, heads=heads, max_kv_len=T)
    assert torch.equal(a, b)
    # an index outside the cache: that row is NaN, the others are untouched by it
    bad = idx_d.clone()
    bad[3, 0] = n_kv
    ops.dec_attn_gather_fwd(q, k, v, bad, len_d, out, heads=heads, max_kv_len=T)
    assert torch.isnan(out[3].float()).all() and not torch.isnan(out[4].float()).any()


@pytest.mark.parametrize("beam", [1, 3, 16])
def test_select_matches_restatement_over_steps(beam):
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(beam)
    n_cap, T, eos = 7, 6, 2
    R = n_cap * beam
    score = -5 * torch.rand(R, generator=gen)
    score[1::max(beam, 2)] = float("-inf")                 # beams not yet alive
    fin = (torch.rand(R, generator=gen) < 0.3).int()
    fin[score == float("-inf")] = 0
    length = torch.randint(1, 3, (R,), generator=gen).int() * fin
    hist = torch.randint(0, 50, (R, T), generator=gen).int()
    anc = torch.randint(0, R, (R, T), generator=gen).int()
    slabs = [torch.zeros(R * T + 3 * R, dtype=torch.int32, device=DEV) for _ in range(2)]
    ancs = [torch.zeros(R * T, dtype=torch.int32, device=DEV) for _ in range(2)]
    from hero_b200.tvc import _beam_state
    cur = torch.cat([hist.view(-1), score.view(torch.int32), fin, length]).to(DEV)
    cur_anc = anc.view(-1).to(DEV)
    ids = torch.empty(R, dtype=torch.int32, device=DEV)
    for step in range(T):
        logp = -3 * torch.rand(R, beam, generator=gen)
        logp = logp.sort(dim=1, descending=True).values
        cols = torch.randint(0, 50, (R, beam), generator=gen).int()
        cols[:, 0][torch.rand(R, generator=gen) < 0.2] = eos
        state_in = _beam_state(cur, R, T)
        if step == 1:
            # planted ties: every candidate of a parent ties with its siblings, and parents 0 and
            # 1 of each caption are live at equal scores, so their candidates tie across parents
            logp[:, :] = -1.0
            if beam > 1:
                sc, fn = state_in[0].view(n_cap, beam), state_in[1].view(n_cap, beam)
                sc[:, 1] = sc[:, 0]
                fn[:, :2] = 0
        lp_d, cl_d = logp.to(DEV), cols.to(DEV)
        want = fake_beam_ops.select_ref(lp_d, cl_d, *state_in, cur_anc, beam=beam, step=step,
                                        max_step=T, eos=eos)
        out, out_anc = slabs[step % 2], ancs[step % 2]
        ops.beam_select(lp_d, cl_d, state_in, cur_anc, _beam_state(out, R, T), out_anc, ids,
                        beam=beam, step=step, max_step=T, eos=eos)
        s, f, ln, h = (x.cpu() for x in _beam_state(out, R, T))
        assert torch.equal(s, want[0]) and torch.equal(f, want[1]) and torch.equal(ln, want[2])
        assert torch.equal(h.view(R, T)[:, :step + 1], want[3][:, :step + 1])
        w = min(step + 2, T)
        assert torch.equal(out_anc.cpu().view(R, T)[:, :w], want[4][:, :w])
        assert torch.equal(ids.cpu(), want[5])
        cur, cur_anc = out, out_anc


def test_tiny_fixture_matches_reference_beam_search(tmp_path, monkeypatch):
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    tx, g = cpu.fixture(), beam_cpu.golden()
    model = cpu.tvc_model(tmp_path, tx).to(DEV)
    gen = beam_cpu.generator(model, tx)
    seen = beam_cpu.recording(monkeypatch)
    thr = beam_cpu.logits_bound(tx)
    for beam in (1, 3, 5):
        seen.clear()
        gen.beam_ids(synth.to_device(attach_plan(cpu.tvc_batch(tx, "val")), DEV), beam)
        compared = beam_cpu.beam_agreement(seen, g, beam, thr)
        print(f"tiny fixture, B = {beam}: {compared} (caption, step) pairs compared")
        assert compared > 0


def _real(seed=3):
    model, path = tvc_gpu._tvc_model(seed=seed)
    return model.to(DEV).eval(), path


def _forced_logprobs(model, batch, ids, bos, n_valid):
    """log-softmax over the first n_valid columns of our teacher-forced logits with the ids as
    the captions: [N, T, n_valid] fp32."""
    n, t = ids.shape
    b = dict(batch)
    b["cap_input_ids"] = torch.cat([torch.full((n, 1), bos, dtype=torch.long),
                                    ids[:, :-1].long()], 1).to(DEV)
    b["cap_pos_ids"] = torch.arange(t).unsqueeze(0).to(DEV)
    with torch.no_grad():
        z = model(b, compute_loss=False).float()
    return torch.log_softmax(z[..., :n_valid], dim=-1)


def test_real_dimensions_greedy_reference_and_scores(monkeypatch):
    import tools.gen_tvc_beam_golden as gb
    from hero_b200 import synth
    from hero_b200.tvc import TvcGenerator
    VideoModelConfig, _ = qa_gpu._reference_module()
    from model.tvc import HeroForTvc as RefTvc
    model, path = _real()
    T, eos = 20, synth.EOS
    hb = synth.syn_tvc_batch(n_videos=4, seed=9, vocab=50265, split="val")
    gen = TvcGenerator(model, T, synth.BOS, eos, fp16=False)
    db = lambda: synth.to_device(hb, DEV)   # noqa: E731
    # B = 1 is greedy decoding, bit for bit up to the first EOS
    greedy = gen.decode_ids(db())
    ids1, _ = gen.beam_ids(db(), 1)
    for g_row, b_row in zip(greedy.tolist(), ids1.tolist()):
        n = g_row.index(eos) + 1 if eos in g_row else T
        assert g_row[:n] == b_row[:n]
    assert gen.beam_search(db(), 1) == gen.greedy_decode(db())
    # B = 5 against the same beam search over the reference in fp32
    B = 5
    ids, score = gen.beam_ids(db(), B)
    seen = []
    ref = RefTvc(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(model.state_dict())
    ref = ref.to(DEV).eval()
    N = ids.shape[0]
    fe = model.v_encoder.f_encoder
    n_valid = fe.embeddings.word_embeddings.weight.shape[0] - fe.vocab_pad
    with torch.no_grad():
        want = gb.beam_search(gb.reference_last_logits(ref, db(), B), N, B, T, synth.BOS, eos,
                              n_valid)
        # our own error on these captions: teacher-forced logits against the reference's
        lp = _forced_logprobs(model, db(), ids, synth.BOS, n_valid)
        inp = torch.cat([torch.full((N, 1), synth.BOS, dtype=torch.long), ids[:, :-1].long()],
                        1).to(DEV)
        enc = ref.encode(db())
        zr = ref.decode(enc, db()["cap_attn_mask"], inp, torch.arange(T).unsqueeze(0).to(DEV),
                        None, compute_loss=False)[..., :n_valid].float()
        lr = torch.log_softmax(zr, dim=-1)
    err = float((lp - lr).abs().max())
    thr = 2 * err
    # the hypotheses kept after each step, as in the tiny-fixture comparison
    from hero_b200 import ops
    select = ops.beam_select

    def spy(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, **kw):
        select(logp, cols, state_in, anc_in, state_out, anc_out, next_ids, **kw)
        seen.append(state_out[3].view(-1, T)[:, :kw["step"] + 1].cpu().clone())
    monkeypatch.setattr(ops, "beam_select", spy)
    gen.beam_ids(db(), B)
    g = {f"b{B}_steps": want["steps"], f"b{B}_margin": want["margin"]}
    compared = beam_cpu.beam_agreement(seen, g, B, thr)
    print(f"real dimensions, B = {B}: log-prob max error {err:.4f}, {compared} (caption, step) "
          f"pairs compared with the reference (margin > {thr:.4f})")
    assert compared > 0
    # each score is the sum of its tokens' log-probabilities under our teacher-forced forward
    tok = lp.gather(2, ids.long().to(DEV)[..., None])[..., 0].cpu().double()
    per_tok = []
    for n in range(N):
        row = ids[n].tolist()
        m = row.index(eos) + 1 if eos in row else T
        per_tok.append(abs(float(score[n]) - float(tok[n, :m].sum())) / m)
    print(f"score vs teacher-forced sum of log-probabilities: max {max(per_tok):.2e} per token")
    # the same kernels on the same rows: 1.4e-6 per token was observed on the H100
    assert max(per_tok) <= 1e-4


def test_beam_search_makes_one_copy_and_no_sync():
    from torch.profiler import ProfilerActivity, profile
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    from hero_b200.tvc import TvcGenerator
    model, _ = tvc_gpu._tvc_model(layers=(2, 2, 2), hidden=256, heads=4, vocab=1000)
    model = model.to(DEV).eval()
    b = attach_plan(synth.syn_tvc_batch(n_videos=8, seed=4, vfeat_dim=64, vocab=1000,
                                        split="val"))
    gen = TvcGenerator(model, 30, synth.BOS, synth.EOS, fp16=False)
    first = gen.beam_search(synth.to_device(b, DEV), 4)    # warm-up (allocations, weight mirror)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gen.beam_search(synth.to_device(b, DEV), 4)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert out == first and len(out) == len(b["clip_ids"])
    db = synth.to_device(b, DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gen.beam_search(db, 4)
        torch.cuda.synchronize()
    d2h = [e for e in prof.events() if "Memcpy DtoH" in e.name]
    assert len(d2h) == 1, [e.name for e in d2h]
