"""TVC early stop (TvcGenerator(early_stop=True)) with hero_b200.ops routed through
tests/fake_early_stop_ops.py, on the tiny fixture tvc_tiny.npz: the argument checks, and for greedy
decoding, beam search (B = 1, 3) and sampling the output rules against early_stop=False when every
row ends at the same step, when rows end at different steps and when no row ends. The kernel and
the loops on the device are covered by test_tvc_early_stop_gpu.py."""
import numpy as np
import pytest
import torch

from tests import fake_early_stop_ops as fes
from tests import test_tvc_cpu as tvc
from tests import test_tvc_decode_ctl_cpu as ctl_cpu

STRATEGIES = ["greedy", "beam1", "beam3", "sample"]
FORCED = 1e3                # an EOS bias no other logit comes near


class EosBias:
    """Sets the LM-head bias of EOS to its initial value + b (the flat buffer's bf16 mirror is
    refreshed on the next pass: the parameter's version changes)."""

    def __init__(self, model, eos):
        self.bias = model.v_encoder.f_encoder.lm_head.bias
        self.eos = eos
        self.base = float(self.bias.detach()[eos])

    def __call__(self, b):
        with torch.no_grad():
            self.bias[self.eos] = self.base + b


def decode(gen, strategy, batch, length_penalty=0.0):
    """The strategy's full output: (ids,) or (ids, score)."""
    if strategy == "greedy":
        return (gen.decode_ids(batch),)
    if strategy.startswith("beam"):
        return gen.beam_ids(batch, int(strategy[4:]), length_penalty)
    return (gen.sample_ids(batch, top_p=0.9, seed=5),)


def first_eos(ids, eos):
    return [r.index(eos) if eos in r else None for r in ids.tolist()]


def check_rules(strategy, full, early, eos, cut_eos):
    """The output rules of early stop against the early_stop=False output. Returns the step after
    which every row has ended, from the full output (greedy / sampling), or None."""
    if strategy.startswith("beam"):
        assert all(torch.equal(a, b) for a, b in zip(full, early)), strategy
        return None
    full, early = full[0], early[0]
    assert [cut_eos(r) for r in full.tolist()] == [cut_eos(r) for r in early.tolist()]
    ends = first_eos(full, eos)
    if None in ends:
        assert torch.equal(early, full), strategy
        return None
    stop = max(ends)
    assert torch.equal(early[:, :stop + 1], full[:, :stop + 1]), strategy
    assert (early[:, stop + 1:] == eos).all(), strategy
    return stop


class Calls(list):
    """The steps of the ops.dec_finished calls of a decode call (one per step the host enqueued)
    and the device stop step of the last one."""
    dev = None

    def stop_step(self):
        from hero_b200 import ops
        if self.dev is None or int(self.dev) == ops.DEC_STOP_UNSET:
            return None
        return int(self.dev)


def counted(monkeypatch):
    from hero_b200 import ops
    calls = Calls()
    inner = ops.dec_finished

    def spy(ids, fin, stop_dev, stop_host, **kw):
        calls.append(kw["step"])
        calls.dev = stop_dev
        inner(ids, fin, stop_dev, stop_host, **kw)
    monkeypatch.setattr(ops, "dec_finished", spy)
    return calls


def generators(model, max_step, **kw):
    from hero_b200 import synth
    from hero_b200.tvc import TvcGenerator
    return (TvcGenerator(model, max_step, synth.BOS, synth.EOS, False, **kw),
            TvcGenerator(model, max_step, synth.BOS, synth.EOS, False, early_stop=True, **kw))


def mixed_bias(strategy, gens, batch, eos, calls, set_bias, length_penalty=0.0):
    """The first EOS bias on a grid under which every row ends, at no fewer than two distinct
    steps, and a stop step is recorded; (bias, full output, early output)."""
    full_gen, early_gen = gens
    # fine below 2 (a decoder initialised at std 0.02 has logits within about +-1), coarse above
    biases = np.round(np.concatenate([np.arange(0.0, 2.0, 0.05), np.arange(2.0, 12.0, 0.25)]),
                      2).tolist()
    for b in biases:
        set_bias(b)
        calls.clear()
        calls.dev = None
        early = decode(early_gen, strategy, batch, length_penalty)
        ends = first_eos(early[0], eos)
        if None not in ends and len(set(ends)) >= 2 and calls.stop_step() is not None:
            return b, decode(full_gen, strategy, batch, length_penalty), early
    raise AssertionError(f"{strategy}: no EOS bias in {biases} ends rows at mixed steps")


@pytest.mark.parametrize("strategy", STRATEGIES)
@pytest.mark.parametrize("case", ["all_end", "mixed", "never_end"])
def test_output_rules(tmp_path, monkeypatch, strategy, case):
    from hero_b200 import synth
    fes.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    batch = tvc.tvc_batch(tx, "val")
    T = ctl_cpu.config()["max_step"]
    eos = synth.EOS
    bias = EosBias(model, eos)
    calls = counted(monkeypatch)
    m = 4
    gens = generators(model, T, min_length=m if case == "all_end" else 0)
    if case == "mixed":
        b, full, early = mixed_bias(strategy, gens, batch, eos, calls, bias)
        print(f"{strategy}: EOS bias {b}, first EOS steps {first_eos(early[0], eos)}")
    else:
        bias(FORCED if case == "all_end" else -FORCED)
        full = decode(gens[0], strategy, batch)
        calls.clear()
        early = decode(gens[1], strategy, batch)
    stop = check_rules(strategy, full, early, eos, gens[0].cut_eos)
    ends = first_eos(early[0], eos)
    if case == "all_end":
        assert ends == [m] * len(ends)
        # the host sees the word as soon as it is written here, so it enqueues up to the stop step
        assert calls == list(range(m + 1))
    elif case == "mixed":
        assert len(set(ends)) >= 2 and calls == list(range(calls.stop_step() + 1))
        assert stop is None or stop == calls.stop_step()
    else:
        assert ends == [None] * len(ends) and calls == list(range(T))
        assert calls.stop_step() is None
    # the same generator without early stop calls no dec_finished
    calls.clear()
    decode(gens[0], strategy, batch)
    assert calls == []


def test_beam_search_with_length_penalty(tmp_path, monkeypatch):
    """Beam search ending mid-loop, with a length penalty: the scores and lengths behind the choice
    are those of the full run, so the chosen beams are too."""
    from hero_b200 import synth
    fes.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    batch = tvc.tvc_batch(tx, "val")
    T = ctl_cpu.config()["max_step"]
    EosBias(model, synth.EOS)(4.0)
    calls = counted(monkeypatch)
    full_gen, early_gen = generators(model, T, no_repeat_ngram_size=2)
    for lp in (0.0, 1.0, 2.5):
        calls.clear()
        early = decode(early_gen, "beam3", batch, lp)
        assert len(calls) < T
        full = decode(full_gen, "beam3", batch, lp)
        assert all(torch.equal(a, b) for a, b in zip(full, early)), lp


def test_early_stop_must_be_a_bool(tmp_path):
    from hero_b200 import synth
    from hero_b200.tvc import TvcGenerator
    model = tvc.tvc_model(tmp_path, tvc.fixture())
    for bad in (1, 0, "yes", None, np.bool_(True)):
        with pytest.raises(ValueError, match="early_stop"):
            TvcGenerator(model, 10, synth.BOS, synth.EOS, False, early_stop=bad)
    for ok in (True, False):
        assert TvcGenerator(model, 10, synth.BOS, synth.EOS, False, early_stop=ok).early_stop is ok


def test_decode_tvc_early_stop_records(tmp_path, monkeypatch):
    from hero_b200 import evalpass, synth
    fes.install(monkeypatch)
    tx = tvc.fixture()
    model = tvc.tvc_model(tmp_path, tx)
    EosBias(model, synth.EOS)(4.0)
    c = ctl_cpu.config()
    batches = [synth.syn_tvc_batch(**dict(c["batch_args"], seed=21 + i), split="val")
               for i in range(2)]
    kw = dict(max_step=c["max_step"], bos=synth.BOS, eos=synth.EOS, tokenizer=tvc._Stub())
    for extra in (dict(), dict(beam_size=3, length_penalty=1.0), dict(do_sample=True, seed=3)):
        want = evalpass.decode_tvc(model, batches, **kw, **extra)
        assert evalpass.decode_tvc(model, batches, early_stop=True, **kw, **extra) == want
    with pytest.raises(ValueError, match="early_stop"):
        evalpass.decode_tvc(model, batches, early_stop="on", **kw)


def test_dec_finished_checks_before_launch():
    """The wrapper and the restatement refuse a negative row count or step, a host word that is not
    pinned host int32 memory, and too few flags, before anything runs."""
    from hero_b200 import ops
    fin = torch.zeros(4, dtype=torch.int32)
    ids = torch.zeros(4, dtype=torch.int32)
    dev = torch.full((1,), ops.DEC_STOP_UNSET, dtype=torch.int32)
    word = torch.full((1,), -1, dtype=torch.int32)          # pageable
    for f in (ops.dec_finished, fes.dec_finished):
        for kw in (dict(rows=-1), dict(step=-1), dict(rows=1.5), dict(rows=5)):
            with pytest.raises(ValueError, match="dec_finished"):
                f(ids, fin, dev, word, **dict(dict(rows=4, eos=2, step=0), **kw))
        for host in (torch.full((1,), -1, dtype=torch.int64), torch.empty(0, dtype=torch.int32),
                     np.full(1, -1, np.int32)):
            with pytest.raises(ValueError, match="stop_host"):
                f(ids, fin, dev, host, rows=4, eos=2, step=0)
    # the wrapper needs a pinned word (only pinned memory has a device mapping)
    with pytest.raises(ValueError, match="pinned"):
        ops.dec_finished(ids, fin, dev, word, rows=4, eos=2, step=0)
    assert (fin == 0).all() and int(dev) == ops.DEC_STOP_UNSET and int(word) == -1


def test_restatement_records_the_first_step_once():
    from hero_b200 import ops
    eos = 2
    fin = torch.zeros(3, dtype=torch.int32)
    dev = torch.full((1,), ops.DEC_STOP_UNSET, dtype=torch.int32)
    word = torch.full((1,), -1, dtype=torch.int32)
    steps = [[5, 2, 7], [2, 9, 9], [4, 4, 4], [4, 4, 2], [9, 9, 9]]
    for t, row in enumerate(steps):
        fes.dec_finished(torch.tensor(row, dtype=torch.int32), fin, dev, word, rows=3, eos=eos,
                         step=t)
        want = -1 if t < 3 else 3
        assert int(word) == want and int(dev) == (ops.DEC_STOP_UNSET if want < 0 else want)
    assert fin.tolist() == [1, 1, 1]
    # beam form: flags read as-is; rows == 0 counts as every row ended
    for rows, flags, want in ((2, [1, 0], -1), (2, [1, 1], 7), (0, [], 7)):
        dev.fill_(ops.DEC_STOP_UNSET)
        word.fill_(-1)
        fes.dec_finished(None, torch.tensor(flags, dtype=torch.int32), dev, word, rows=rows,
                         eos=eos, step=7)
        assert int(word) == want and int(dev) == (ops.DEC_STOP_UNSET if want < 0 else want)
