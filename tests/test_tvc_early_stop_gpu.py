"""TVC early stop on the H100: hero_dec_finished against its restatement
(tests/fake_early_stop_ops.py) in both forms at 0, 1, 35 and 1600 rows, the stop step recorded once
and mirrored into the pinned host word, the bounds refused with nothing launched; on a small
decoder, greedy decoding, beam search (B = 1, 3, 5, with and without a length penalty) and sampling
against early_stop=False when every row ends at one step, at mixed steps and never, with and
without n-gram blocking; a loop that ends at step 0 of 1023 launching less than half of the full
loop; no host synchronisation and one device->host copy per call; and decode_tvc's records at real
dimensions."""
import pytest
import torch

from tests import fake_early_stop_ops as fes
from tests import test_tvc_early_stop_cpu as es_cpu
from tests import test_tvc_gpu as tvc_gpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
EOS = 2


def _word():
    return torch.full((1,), -1, dtype=torch.int32).pin_memory()


def _state(rows, device):
    from hero_b200 import ops
    return (torch.zeros(rows, dtype=torch.int32, device=device),
            torch.full((1,), ops.DEC_STOP_UNSET, dtype=torch.int32, device=device))


@pytest.mark.parametrize("rows", [1, 35, 1600, 0])
@pytest.mark.parametrize("form", ["ids", "flags"])
def test_dec_finished_matches_restatement(rows, form):
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(rows)
    T = 12
    # row r ends at step end[r] (ids form: emits EOS there, other tokens before and after; flags
    # form: its flag is set from then on); the last row to end does so at step 7
    end = torch.randint(0, 8, (rows,), generator=gen)
    if rows:
        end[rows // 2] = 7
    fin, dev = _state(rows, DEV)
    fin_r, dev_r = _state(rows, "cpu")
    word, word_r = _word(), torch.full((1,), -1, dtype=torch.int32)
    want_stop = 7 if rows else 0
    for t in range(T):
        if form == "ids":
            ids = torch.randint(3, 50, (rows,), generator=gen, dtype=torch.int32)
            ids[end == t] = EOS
            if t > 9:
                ids[:] = 5                                   # no EOS: the flags stay set
            ops.dec_finished(ids.to(DEV), fin, dev, word, rows=rows, eos=EOS, step=t)
            fes.dec_finished(ids, fin_r, dev_r, word_r, rows=rows, eos=EOS, step=t)
        else:
            flags = (end <= t).int()
            if t > 9:
                flags[:rows // 3] = 0                        # a set step is never moved
            fin.copy_(flags.to(DEV))
            ops.dec_finished(None, fin, dev, word, rows=rows, eos=EOS, step=t)
            fes.dec_finished(None, flags, dev_r, word_r, rows=rows, eos=EOS, step=t)
            fin_r = flags
        torch.cuda.synchronize()
        assert torch.equal(fin.cpu(), fin_r), (form, rows, t)
        assert int(dev) == int(dev_r) and int(word) == int(word_r), (form, rows, t)
        assert int(word) == (want_stop if t >= want_stop else -1), (form, rows, t)
        assert int(dev) == (want_stop if t >= want_stop else ops.DEC_STOP_UNSET)


def test_dec_finished_refuses_with_nothing_launched():
    from hero_b200 import ops
    fin, dev = _state(4, DEV)
    ids = torch.full((4,), EOS, dtype=torch.int32, device=DEV)
    word = _word()
    torch.cuda.synchronize()
    n = ops.launch_count()
    with pytest.raises(ValueError, match="rows"):
        ops.dec_finished(ids, fin, dev, word, rows=-1, eos=EOS, step=0)
    for host in (torch.full((1,), -1, dtype=torch.int32),                 # pageable
                 torch.full((1,), -1, dtype=torch.int32, device=DEV),     # device memory
                 torch.full((1,), -1, dtype=torch.int64).pin_memory()):
        with pytest.raises(ValueError, match="pinned"):
            ops.dec_finished(ids, fin, dev, host, rows=4, eos=EOS, step=0)
    torch.cuda.synchronize()
    assert ops.launch_count() == n
    assert (fin == 0).all() and int(dev) == ops.DEC_STOP_UNSET and int(word) == -1
    ops.dec_finished(ids, fin, dev, word, rows=4, eos=EOS, step=3)            # and it does run
    torch.cuda.synchronize()
    assert (fin == 1).all() and int(dev) == 3 and int(word) == 3


# ------------------------------------------------------------------ decode loops
def _small():
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    model, _ = tvc_gpu._tvc_model(layers=(2, 2, 2), hidden=256, heads=4, vocab=1000)
    model = model.to(DEV).eval()
    b = attach_plan(synth.syn_tvc_batch(n_videos=8, seed=4, vfeat_dim=64, vocab=1000,
                                        split="val"))
    return model, b


STRATEGIES = ["greedy", "beam1", "beam3", "beam5", "sample"]


@pytest.mark.parametrize("ngram", [0, 3])
@pytest.mark.parametrize("case", ["all_end", "mixed", "never_end"])
def test_output_rules(tmp_path, monkeypatch, case, ngram):
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    from tests import test_tvc_cpu as tvc_cpu
    model, b = _small()
    T, m = 30, 6
    if case == "mixed":
        # the small decoder, initialised at std 0.02, decodes nearly the same tokens for every
        # caption; the tiny fixture's (std 0.1) captions differ enough to end at mixed steps
        tx = tvc_cpu.fixture()
        model = tvc_cpu.tvc_model(tmp_path, tx).to(DEV)
        b = attach_plan(tvc_cpu.tvc_batch(tx, "val"))
        T = es_cpu.ctl_cpu.config()["max_step"]
    bias = es_cpu.EosBias(model, EOS)
    calls = es_cpu.counted(monkeypatch)
    gens = es_cpu.generators(model, T, min_length=m if case == "all_end" else 0,
                             no_repeat_ngram_size=ngram)
    db = synth.to_device(b, DEV)
    for strategy in STRATEGIES:
        for lp in ((0.0, 1.0) if strategy.startswith("beam") else (0.0,)):
            calls.clear()
            calls.dev = None
            if case == "mixed":
                _, full, early = es_cpu.mixed_bias(strategy, gens, db, EOS, calls, bias, lp)
            else:
                bias(es_cpu.FORCED if case == "all_end" else -es_cpu.FORCED)
                full = es_cpu.decode(gens[0], strategy, db, lp)
                early = es_cpu.decode(gens[1], strategy, db, lp)
            stop = es_cpu.check_rules(strategy, full, early, EOS, gens[0].cut_eos)
            ends = es_cpu.first_eos(early[0], EOS)
            got = calls.stop_step()
            print(f"{case}, n-gram {ngram}, {strategy}, length penalty {lp}: device stop {got}, "
                  f"{len(calls)} of {T} steps enqueued, first EOS steps "
                  f"{sorted(set(ends), key=str)}")
            # the host enqueued every step up to the device's stop step, and perhaps a few more
            assert calls == list(range(len(calls)))
            if case == "all_end":
                assert ends == [m] * len(ends) and got == m and len(calls) > m
            elif case == "mixed":
                assert len(set(ends)) >= 2 and got is not None and len(calls) > got
                assert stop is None or stop == got
            else:
                assert ends == [None] * len(ends) and got is None and len(calls) == T


def test_it_stops_early():
    """EOS forced at step 0 with max_step 1023: the host stops enqueueing long before the end. The
    bound is loose: how many steps the host runs ahead of the device depends on the machine."""
    from hero_b200 import ops, synth
    model, b = _small()
    es_cpu.EosBias(model, EOS)(es_cpu.FORCED)
    full_gen, early_gen = es_cpu.generators(model, 1023)
    db = synth.to_device(b, DEV)
    for strategy in ("greedy", "beam5", "sample"):
        counts, outs = [], []
        for gen in (full_gen, early_gen):
            es_cpu.decode(gen, strategy, db)                    # warm-up
            torch.cuda.synchronize()
            ops.reset_launch_count()
            outs.append(es_cpu.decode(gen, strategy, db))
            counts.append(ops.launch_count())
        print(f"{strategy}: {counts[0]} launches without early stop, {counts[1]} with")
        assert counts[1] < counts[0] / 2, (strategy, counts)
        es_cpu.check_rules(strategy, outs[0], outs[1], EOS, full_gen.cut_eos)


@pytest.mark.parametrize("forced", [False, True])
def test_no_sync_and_one_copy(forced):
    from torch.profiler import ProfilerActivity, profile
    from hero_b200 import synth
    from hero_b200.tvc import TvcGenerator
    model, b = _small()
    if forced:
        es_cpu.EosBias(model, EOS)(es_cpu.FORCED)
    gen = TvcGenerator(model, 30, synth.BOS, synth.EOS, fp16=False, min_length=4,
                       early_stop=True)
    calls = {"greedy": lambda d: gen.greedy_decode(d), "beam": lambda d: gen.beam_search(d, 5),
             "sample": lambda d: gen.sample(d, temperature=0.9, top_p=0.9, seed=7)}
    for name, call in calls.items():
        first = call(synth.to_device(b, DEV))                 # warm-up
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = call(synth.to_device(b, DEV))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert out == first and len(out) == len(b["clip_ids"]), name
        if forced:
            assert all(len(r) == 4 for r in out), name
        db = synth.to_device(b, DEV)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(db)
            torch.cuda.synchronize()
        d2h = [e for e in prof.events() if "Memcpy DtoH" in e.name]
        assert len(d2h) == 1, (name, [e.name for e in d2h])


def test_decode_tvc_records_real_dimensions():
    """decode_tvc on syn_tvc_val batches at real dimensions (6 + 3 encoder layers, 2 decoder
    layers, H 768, vocabulary 50 272): the same records with and without early stop, every
    strategy, with every caption ending at step 5 and with no caption ending."""
    from hero_b200 import evalpass, synth
    from tests import test_tvc_cpu as tvc_cpu
    model, _ = tvc_gpu._tvc_model(seed=3)
    model = model.to(DEV).eval()
    bias = es_cpu.EosBias(model, EOS)
    loader = [synth.to_device(synth.syn_tvc_val(seed=s), DEV) for s in range(2)]
    kw = dict(max_step=30, bos=synth.BOS, eos=synth.EOS, tokenizer=tvc_cpu._Stub())
    for b, extra in ((es_cpu.FORCED, dict(min_length=5)), (-es_cpu.FORCED, dict())):
        bias(b)
        for strategy in (dict(), dict(beam_size=5, length_penalty=1.0),
                         dict(do_sample=True, top_p=0.9, seed=1)):
            want = evalpass.decode_tvc(model, loader, **kw, **extra, **strategy)
            got = evalpass.decode_tvc(model, loader, early_stop=True, **kw, **extra, **strategy)
            assert got == want, strategy
            if b > 0:
                assert all(len(r["descs"][0]["desc"].split()) == 5 for r in got)
