"""TVC decoding controls (TvcGenerator's no_repeat_ngram_size / min_length, and sampling) with
hero_b200.ops routed through tests/fake_decode_ctl_ops.py, on the tiny fixture tvc_tiny.npz: the ban
restatement against a brute-force enumeration of n-grams, the caption properties under greedy, beam
and sampled decoding, greedy decoding against a plain loop over the model's own masked logits,
defaults that change nothing, sampling's determinism, the bounds, and the evaluation records on one
process and on gloo ranks. The kernels are covered by test_tvc_decode_ctl_gpu.py."""
import inspect
import json
import math
import os
import socket
import tempfile
from collections import Counter
from pathlib import Path

import pytest
import torch
import torch.multiprocessing as mp

from tests import fake_decode_ctl_ops as fdc
from tests import test_tvc_cpu as tvc


def config():
    return json.loads(str(tvc.fixture()["config"]))


def generator(model, **kw):
    from hero_b200 import synth
    from hero_b200.tvc import TvcGenerator
    return TvcGenerator(model, config()["max_step"], synth.BOS, synth.EOS, False, **kw)


def brute_force_bans(s, n):
    """Tokens that would complete an n-gram of s already present in s (enumerated as tuples)."""
    if n < 1 or len(s) < n:
        return set()
    follow = {}
    for j in range(len(s) - n + 1):
        follow.setdefault(tuple(s[j:j + n - 1]), set()).add(s[j + n - 1])
    return follow.get(tuple(s[len(s) - n + 1:]), set())


def planted_history(rows, steps, vocab, gen):
    """Random histories over a small alphabet with a copied stretch, so repeats are common."""
    h = torch.randint(3, 3 + vocab, (rows, steps), generator=gen)
    for r in range(rows):
        if steps >= 6:
            a = int(torch.randint(0, steps // 2, (1,), generator=gen))
            ln = int(torch.randint(2, steps // 2 + 1, (1,), generator=gen))
            b = min(steps, a + ln + int(torch.randint(0, 3, (1,), generator=gen)))
            k = min(ln, steps - b)
            h[r, b:b + k] = h[r, a:a + k].clone()
    return h.int()


@pytest.mark.parametrize("layout", ["greedy", "beam"])
def test_ban_restatement_equals_brute_force(layout):
    gen = torch.Generator().manual_seed(3)
    rows, T, V, bos, eos = 6, config()["max_step"], 40, 0, 2
    for n in range(1, 5):
        for alphabet in (3, 6):
            h = planted_history(rows, T, alphabet, gen)
            if layout == "greedy":          # out [T + 1, rows], out[0] = bos, history out[1:]
                out = torch.cat([torch.full((1, rows), bos, dtype=torch.int32), h.t()], 0)
                hist, steps, rs = out[1:], rows, 1
            else:                           # beam-state slab: row r, step j at hist[r * T + j]
                hist, steps, rs = h.reshape(-1).clone(), 1, T
            for t in range(T):
                for min_len in (0, 3):
                    x = torch.randn(rows, V + 8)
                    x0 = x.clone()
                    fdc.ban_tokens(x, V, hist, step_stride=steps, row_stride=rs, bos=bos, step=t,
                                   ngram=n, min_length=min_len, eos=eos)
                    for r in range(rows):
                        s = [bos] + h[r, :t].tolist()
                        want = {c for c in brute_force_bans(s, n) if c < V}
                        if t < min_len:
                            want.add(eos)
                        got = set(torch.nonzero(x[r] != x0[r]).flatten().tolist())
                        assert got == want, (layout, n, t, r)
                        assert (x[r, sorted(got)] == -math.inf).all()


def has_repeat(seq, n):
    grams = [tuple(seq[j:j + n]) for j in range(len(seq) - n + 1)]
    return len(grams) != len(set(grams))


def check_properties(rows, n, min_len, eos, bos):
    for row in rows:
        row = list(row)
        cut = row[:row.index(eos) + 1] if eos in row else row
        assert not has_repeat([bos] + cut, n), cut
        assert eos not in row[:min_len], row


def test_captions_obey_the_controls(tmp_path, monkeypatch):
    from hero_b200 import synth
    fdc.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    b = tvc.tvc_batch(tx, "val")
    gen = generator(model, no_repeat_ngram_size=2, min_length=3)
    plain = generator(model)
    ids = {"greedy": gen.decode_ids(b), "beam": gen.beam_ids(b, 3)[0],
           "sample": gen.sample_ids(b, seed=5), "sample_p": gen.sample_ids(b, top_p=0.8, seed=6)}
    for name, v in ids.items():
        check_properties(v.tolist(), 2, 3, synth.EOS, synth.BOS)
    # the controls are not vacuous here: without them greedy decoding repeats or stops early
    raw = plain.decode_ids(b).tolist()
    assert any(has_repeat([synth.BOS] + r, 2) or synth.EOS in r[:3] for r in raw)
    assert ids["greedy"].tolist() != raw


def test_greedy_with_controls_equals_a_plain_loop(tmp_path, monkeypatch):
    """Greedy ids with the controls on equal, step by step, the argmax of the model's own
    teacher-forced logits masked by the brute-force rules (where the top-2 gap is clear)."""
    from hero_b200 import synth
    fdc.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    n, min_len = 2, 4
    ids = generator(model, no_repeat_ngram_size=n, min_length=min_len).decode_ids(
        tvc.tvc_batch(tx, "val"))
    N, T = ids.shape
    b = tvc.tvc_batch(tx, "val")
    b["cap_input_ids"] = torch.cat([torch.full((N, 1), synth.BOS, dtype=torch.long),
                                    ids[:, :-1].long()], 1)
    b["cap_pos_ids"] = torch.arange(T).unsqueeze(0)
    with torch.no_grad():
        logits = model(b, compute_loss=False).float().clone()
    compared = 0
    for r in range(N):
        for t in range(T):
            z = logits[r, t].clone()
            s = [synth.BOS] + ids[r, :t].tolist()
            for c in brute_force_bans(s, n):
                z[c] = -math.inf
            if t < min_len:
                z[synth.EOS] = -math.inf
            top = z.topk(2).values
            if top[0] - top[1] > 1e-3:
                assert int(z.argmax()) == int(ids[r, t]), (r, t)
                compared += 1
    assert compared > N * T // 2


def counting(monkeypatch):
    """Wraps every public function of hero_b200.ops so that each call is counted by name."""
    from hero_b200 import ops
    calls = Counter()
    for name, f in list(vars(ops).items()):
        if name.startswith("_") or not inspect.isfunction(f) or "launch_count" in name:
            continue

        def wrap(*a, _f=f, _n=name, **kw):
            calls[_n] += 1
            return _f(*a, **kw)
        monkeypatch.setattr(ops, name, wrap)
    return calls


def test_controls_off_change_nothing(tmp_path, monkeypatch):
    from hero_b200 import ops
    fdc.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    b = tvc.tvc_batch(tx, "val")
    generator(model).decode_ids(b)          # the first call builds the model's flat weights
    calls = counting(monkeypatch)
    runs = []
    for gen in (generator(model), generator(model, min_length=0, no_repeat_ngram_size=0)):
        calls.clear()
        ops.reset_launch_count()
        out = (gen.decode_ids(b), gen.greedy_decode(b)) + gen.beam_ids(b, 3, 1.0) + \
            (gen.beam_search(b, 3),)
        runs.append((out, dict(calls), ops.launch_count()))
    (a, ca, la), (o, co, lo) = runs
    for x, y in zip(a, o):
        assert torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y
    assert ca == co and la == lo and "ban_tokens" not in co
    # with a control on, every step bans (n-gram size 3 from step 2 on, EOS while t < 1)
    calls.clear()
    generator(model, no_repeat_ngram_size=3).decode_ids(b)
    assert calls["ban_tokens"] == config()["max_step"]


def test_every_uniform_lies_strictly_inside_the_unit_interval():
    """All 2^23 values the uniform can take (it keeps the top 23 bits of the hash): 0 < u < 1,
    each one exact and distinct, so every Gumbel variable is finite."""
    top = torch.arange(2 ** 23, dtype=torch.long) << 9
    for low in (0, 511):
        u = fdc.uniform_of_hash(top | low)
        assert u.dtype == torch.float32 and (u > 0).all() and (u < 1).all()
        assert float(u.min()) == 2.0 ** -24 and float(u.max()) == 1.0 - 2.0 ** -24
        assert torch.unique(u).numel() == 2 ** 23
        g = -torch.log(-torch.log(u))
        assert torch.isfinite(g).all() and float(g.max()) < 17.0


def largest_uniform_row(n=50272, seed=123, step=4):
    found = fdc.largest_uniform(n, seed, step)
    assert found is not None
    return found


def test_largest_uniform_cannot_override_the_logits():
    """The column that gets the largest uniform of its row: banned (-inf) it is never drawn, and
    with a logit far below the others it is not drawn either (its Gumbel variable is at most
    16.6); with a logit far above them it is."""
    row, col = largest_uniform_row()
    n = 50272
    x = torch.randn(row + 1, n, generator=torch.Generator().manual_seed(0))
    for kw in (dict(top_k=0, top_p=1.0), dict(top_k=0, top_p=0.999), dict(top_k=n - 1, top_p=1.0)):
        for val, drawn in ((-math.inf, False), (-40.0, False), (40.0, True)):
            x[row, col] = val
            ids, _ = fdc.sample_ref(x, n, temperature=1.0, seed=123, step=4, **kw)
            assert (int(ids[row]) == col) == drawn, (kw, val)


def test_decode_tvc_checks_the_seed(tmp_path, monkeypatch):
    from hero_b200 import evalpass, synth
    from hero_b200.tvc import sampling_seed
    fdc.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    kw = dict(max_step=config()["max_step"], bos=synth.BOS, eos=synth.EOS, tokenizer=tvc._Stub(),
              do_sample=True)
    for bad in (-1, 2 ** 32, 1.5):
        with pytest.raises(ValueError, match="seed"):
            evalpass.decode_tvc(model, [tvc.tvc_batch(tx, "val")], seed=bad, **kw)
        with pytest.raises(ValueError, match="seed"):
            sampling_seed(bad, 0, 0)
    assert 0 <= sampling_seed(2 ** 32 - 1, 1, 2) < 2 ** 32


def test_sampling_is_keyed_and_top_k_1_is_greedy(tmp_path, monkeypatch):
    """top_k=1 keeps every column tied at the maximum and draws among them, where rank_topk takes
    the lowest: the two agree on rows without an exact tie at the top, as on this fixture."""
    fdc.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    b = tvc.tvc_batch(tx, "val")
    gen = generator(model)
    assert gen.sample(b, top_k=1, seed=9) == gen.greedy_decode(b)
    assert gen.sample(b, top_k=1, temperature=0.5, top_p=0.3, seed=1) == gen.greedy_decode(b)
    one = gen.sample_ids(b, seed=11)
    assert torch.equal(gen.sample_ids(b, seed=11), one)
    assert not torch.equal(gen.sample_ids(b, seed=12), one)
    assert gen.sample(b, seed=11) == [gen.cut_eos(r) for r in one.tolist()]


def test_bounds_raise_before_any_op(tmp_path, monkeypatch):
    from hero_b200 import evalpass, ops, synth
    fdc.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)

    def no_encode(batch):
        raise AssertionError("an op ran before the bounds were checked")
    monkeypatch.setattr(model, "encode", no_encode)
    b = tvc.tvc_batch(tx, "val")
    for kw, match in ((dict(no_repeat_ngram_size=-1), "no_repeat_ngram_size"),
                      (dict(no_repeat_ngram_size=1.5), "no_repeat_ngram_size"),
                      (dict(min_length=-2), "min_length")):
        g = generator(model, **kw)
        for call in (g.decode_ids, g.greedy_decode, lambda x: g.beam_ids(x, 3),
                     lambda x: g.sample(x)):
            with pytest.raises(ValueError, match=match):
                call(b)
    g = generator(model)
    for kw, match in ((dict(temperature=0.0), "temperature"), (dict(temperature=-1.0), "temperature"),
                      (dict(temperature=float("nan")), "temperature"),
                      (dict(temperature=float("inf")), "temperature"),
                      (dict(top_k=-1), "top_k"), (dict(top_p=0.0), "top_p"),
                      (dict(top_p=1.5), "top_p"), (dict(top_p=float("nan")), "top_p"),
                      (dict(seed=-1), "seed"), (dict(seed=2 ** 32), "seed")):
        with pytest.raises(ValueError, match=match):
            g.sample_ids(b, **kw)
    monkeypatch.setattr(ops, "SAMPLE_MAX_COLS", 100)          # fewer columns than the vocabulary
    with pytest.raises(ValueError, match="sampling takes at most"):
        g.sample(b)
    # max_step + 2 must not exceed the vocabulary when a control is on
    fe = model.v_encoder.f_encoder
    T = config()["max_step"]
    monkeypatch.setattr(fe, "vocab_pad", fe.embeddings.word_embeddings.weight.shape[0] - (T + 1))
    for kw in (dict(no_repeat_ngram_size=2), dict(min_length=1)):
        g = generator(model, **kw)
        for call in (g.decode_ids, lambda x: g.beam_ids(x, 3), lambda x: g.sample_ids(x)):
            with pytest.raises(ValueError, match="max_step"):
                call(b)
    kw = dict(max_step=T, bos=synth.BOS, eos=synth.EOS, tokenizer=tvc._Stub())
    with pytest.raises(ValueError, match="do_sample"):
        evalpass.decode_tvc(model, [b], beam_size=3, do_sample=True, **kw)


def test_kernel_wrappers_check_bounds_before_launch():
    from hero_b200 import ops
    x = torch.zeros(2, 8)
    h = torch.zeros(2, 4, dtype=torch.int32)
    base = dict(step_stride=2, row_stride=1, bos=0, step=1, ngram=2, min_length=0, eos=2)
    for kw in (dict(ngram=-1), dict(min_length=-1), dict(step=-1), dict(step=1024),
               dict(step=5)):
        with pytest.raises(ValueError, match="ban_tokens"):
            ops.ban_tokens(x, 8, h, **dict(base, **kw))
    with pytest.raises(ValueError, match="ban_tokens"):
        ops.ban_tokens(x, 9, h, **base)
    ids = torch.zeros(2, dtype=torch.int32)
    base = dict(temperature=1.0, top_k=0, top_p=1.0, seed=0, step=0)
    for n, kw in ((0, {}), (9, {}), (8, dict(temperature=0.0)), (8, dict(top_k=-1)),
                  (8, dict(top_p=0.0)), (8, dict(top_p=1.01)), (8, dict(seed=-1)),
                  (8, dict(seed=2 ** 32)), (8, dict(step=-1))):
        with pytest.raises(ValueError, match="sample_tokens"):
            ops.sample_tokens(x, n, ids, **dict(base, **kw))
    big = torch.zeros(1, ops.SAMPLE_MAX_COLS + 1)
    with pytest.raises(ValueError, match="sample_tokens"):
        ops.sample_tokens(big, big.shape[1], ids, **base)


# ------------------------------------------------------------------ evaluation records
def _batches():
    from hero_b200 import synth
    c = config()
    return [synth.syn_tvc_batch(**dict(c["batch_args"], seed=21 + i), split="val")
            for i in range(3)]


SAMPLE_KW = dict(do_sample=True, top_p=0.9, temperature=0.8, seed=77, no_repeat_ngram_size=2,
                 min_length=2)


def _decode(tmp, batches):
    from hero_b200 import evalpass, synth
    tx = tvc.fixture()
    return evalpass.decode_tvc(tvc.tvc_model(tmp, tx), batches, max_step=config()["max_step"],
                               bos=synth.BOS, eos=synth.EOS, tokenizer=tvc._Stub(), **SAMPLE_KW)


def _expected(tmp, batches, rank):
    """Records of rank `rank`'s batches, each sampled under its own key."""
    from hero_b200.tvc import sampling_seed
    model = tvc.tvc_model(tmp, tvc.fixture())
    gen = generator(model, no_repeat_ngram_size=2, min_length=2)
    out = []
    for i, b in enumerate(batches):
        caps = gen.sample(b, top_p=0.9, temperature=0.8, seed=sampling_seed(77, rank, i))
        for vid, cid, ts, ids in zip(b["vid_names"], b["clip_ids"], b["all_ts"], caps):
            out.append({"vid_name": vid, "clip_id": cid, "ts": ts,
                        "descs": [{"desc": " ".join(f"w{i}" for i in ids)}]})
    return out


def test_decode_tvc_sampled_records(tmp_path, monkeypatch):
    fdc.install(monkeypatch)
    batches = _batches()
    recs = _decode(tmp_path, batches)
    assert recs == _expected(tmp_path, batches, 0)
    assert len(recs) == sum(len(b["clip_ids"]) for b in batches)
    # every batch draws from its own uniforms: the same batch twice gives different captions
    twice = _decode(tmp_path, [batches[0], batches[0]])
    k = len(batches[0]["clip_ids"])
    assert twice[:k] == recs[:k] and twice[k:] != twice[:k]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


class _Patch:
    @staticmethod
    def setattr(obj, name, value):
        setattr(obj, name, value)


def _worker(rank, world, port, ret):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    import torch.distributed as dist
    from hero_b200 import distributed as hd
    hd.init(backend="gloo")
    try:
        fdc.install(_Patch)
        with tempfile.TemporaryDirectory() as tmp:
            ret[rank] = _decode(Path(tmp), _batches()[rank::world])
    finally:
        if dist.is_initialized():           # one rank is a single-process job: no group
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2])
def test_decode_tvc_sampling_data_parallel(tmp_path, monkeypatch, world):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    fdc.install(monkeypatch)
    batches = _batches()
    want = [r for rank in range(world)
            for r in _expected(tmp_path, batches[rank::world], rank)]
    assert len(want) == sum(len(b["clip_ids"]) for b in batches)
    for rank in range(world):
        assert ret[rank] == want
