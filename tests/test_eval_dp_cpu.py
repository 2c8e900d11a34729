"""Data-parallel evaluation (hero_b200/evalpass.py with distributed.size() > 1) on gloo, world
sizes 2 and 3, with hero_b200.ops routed through the torch restatements of tests/fake_*_ops.py.

Rank r evaluates batches r::W (queries, clips with their global rows); every rank must return the
same object, and that object must equal the one-process call over the same batches taken in rank
order (rank 0's, then rank 1's, ...), which is the order the gathered lists keep. Counts, ids,
records, submissions and retrieval metrics are compared exactly. Loss / l2 / cosine sums are
compared at 1e-6 relative: the sharded run adds each rank's fp32 sum in fp64, the one-process run
adds the batches in one fp32 accumulator, so the two differ by fp32 summation order only."""
import json
import os
import socket
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from torch import nn

REL = 1e-6
RATES = ("tok_per_s", "feat_per_s", "ex_per_s")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, fn_name, args, ret):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    import torch.distributed as dist
    from hero_b200 import distributed as hd
    hd.init(backend="gloo")
    try:
        ret[rank] = globals()[fn_name](rank, world, *args)
    finally:
        dist.destroy_process_group()


def _run(fn_name, world, *args):
    """fn_name(rank, world, *args) on `world` gloo ranks; returns [result of rank r]."""
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), fn_name, args, ret), nprocs=world, join=True)
    return [ret[r] for r in range(world)]


def _rank_order(items, world):
    return [x for r in range(world) for x in items[r::world]]


class _Patch:
    """monkeypatch stand-in for spawned workers (nothing to undo: the process exits)."""

    @staticmethod
    def setattr(obj, name, value):
        setattr(obj, name, value)


class _StepClock:
    """time.time stand-in that alternates 0.0 and 1.0: every validation reads the clock once
    before and once after its loop, so its wall time is exactly 1 s and each rate equals the
    count it divides (the global count when merged)."""

    def __init__(self):
        self.n = 0

    def __call__(self):
        self.n += 1
        return float((self.n - 1) % 2)


def _close(got, want, rel=REL):
    assert set(got) == set(want)
    for k, v in want.items():
        assert got[k] == pytest.approx(v, rel=rel, abs=1e-12), k


# ------------------------------------------------------------------ sum_over_ranks
def _sum_case(rank, world):
    from hero_b200 import distributed as hd
    out = []
    for dtype in (torch.float32, torch.float64):
        t = torch.tensor([[0.1 * (rank + 1), 2.0 ** 30 + rank], [1e-3, -rank]], dtype=dtype)
        out.append(hd.sum_over_ranks(t))
    try:
        hd.sum_over_ranks(torch.ones(2, dtype=torch.int64))
        out.append(None)
    except TypeError as e:
        out.append(str(e))
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_sum_over_ranks_is_the_rank_order_sum_on_every_rank(world):
    from hero_b200 import distributed as hd
    res = _run("_sum_case", world)
    for i, dtype in enumerate((torch.float32, torch.float64)):
        parts = [torch.tensor([[0.1 * (r + 1), 2.0 ** 30 + r], [1e-3, -r]], dtype=dtype)
                 for r in range(world)]
        want = parts[0].clone()
        for p in parts[1:]:
            want += p
        for r in range(world):
            got = res[r][i]
            assert got.dtype == dtype and got.shape == (2, 2)
            assert torch.equal(got, want)
            assert torch.equal(got.view(-1).view(torch.uint8), res[0][i].view(-1).view(torch.uint8))
    assert all("fp32 / fp64" in res[r][2] for r in range(world))
    t = torch.tensor([1.5, 2.5])
    alone = hd.sum_over_ranks(t)                       # no process group: a copy
    assert torch.equal(alone, t) and alone.data_ptr() != t.data_ptr()


# ------------------------------------------------------------------ pretraining validation
def _pretrain_loaders():
    from tests.test_pretrain_val_cpu import loaders
    return loaders(attach=True)


def _pretrain_case(rank, world, n_batches):
    from hero_b200 import evalpass
    from tests import fake_pretrain_val_ops
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model
    fake_pretrain_val_ops.install(_Patch)
    with tempfile.TemporaryDirectory() as tmp:
        model = build_model(Path(tmp), gu.load("pretrain_val_tiny.npz"))
    ld = {t: bs[:n_batches][rank::world] for t, bs in _pretrain_loaders().items()
          if t != "vsm" or n_batches % world == 0}
    import time
    _Patch.setattr(time, "time", _StepClock())
    return evalpass.validate_pretrain(model, ld, pv.Opts)


# VSM takes its in-batch negatives from every rank's current batch (the model's val_gather_gpus,
# as the reference's forward does), so its ranking losses are not those of the one-process call,
# and every rank must run the same number of VSM batches: it is left out where a rank has none.
# Its span loss is per query and must match.
VSM_NEGATIVES = ("vsm_valid/loss_overall", "vsm_valid/loss_neg_ctx", "vsm_valid/loss_neg_q")


@pytest.mark.parametrize("world, n_batches", [(2, 2), (3, 2), (2, 1)])
def test_validate_pretrain_merges_every_rank(tmp_path, monkeypatch, world, n_batches):
    """(3, 2): rank 2 has no batch of any task; (2, 1): rank 1 has none."""
    from hero_b200 import evalpass
    from tests import fake_pretrain_val_ops
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model
    res = _run("_pretrain_case", world, n_batches)
    fake_pretrain_val_ops.install(monkeypatch)
    model = build_model(tmp_path, gu.load("pretrain_val_tiny.npz"))
    ld = {t: _rank_order(bs[:n_batches], world) for t, bs in _pretrain_loaders().items()
          if t != "vsm" or n_batches % world == 0}
    import time
    monkeypatch.setattr(time, "time", _StepClock())
    want = evalpass.validate_pretrain(model, ld, pv.Opts)
    monkeypatch.undo()
    rates = {k for k in want if k.endswith(RATES)}
    assert len(rates) == len(ld) >= len(pv.TASKS) - 1
    for r in range(world):
        assert set(res[r]) == set(want)
        # a 1 s wall time everywhere: the rate is the global count on every rank
        assert {k: res[r][k] for k in rates} == {k: want[k] for k in rates}
        fixed = {k: v for k, v in res[r].items() if k not in rates}
        assert fixed == {k: v for k, v in res[0].items() if k not in rates}     # bitwise, all ranks
        _close({k: v for k, v in fixed.items() if k not in VSM_NEGATIVES},
               {k: v for k, v in want.items() if k not in rates and k not in VSM_NEGATIVES})
        for k, v in fixed.items():
            if k.endswith("acc"):                      # hit counts / counts: exact
                assert v == want[k], k


def _vsm_unequal_case(rank, world):
    from hero_b200 import evalpass
    from tests import fake_pretrain_val_ops
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model
    fake_pretrain_val_ops.install(_Patch)
    with tempfile.TemporaryDirectory() as tmp:
        model = build_model(Path(tmp), gu.load("pretrain_val_tiny.npz"))
    try:
        evalpass.validate_pretrain(model, {"vsm": _pretrain_loaders()["vsm"][rank:]}, pv.Opts)
    except ValueError as e:
        return str(e)
    return None


def test_validate_vsm_with_unequal_batch_counts_raises_on_every_rank():
    """Rank 0 has two VSM batches, rank 1 one: without the check rank 0 would wait in the
    model's cross-rank gather for a rank that has finished."""
    for msg in _run("_vsm_unequal_case", 2):
        assert msg is not None and "[2, 1] batches" in msg, msg


# ------------------------------------------------------------------ video QA and VIOLIN
class _ScoresOfBatch(nn.Module):
    """Returns the scores stored in the batch, so a batch scores the same on any rank."""

    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(torch.zeros(1))

    def forward(self, batch, task, compute_loss=False):
        assert not compute_loss
        return batch["s"]


def _qa_batches(kind, n_batches, no_gt_batch=None):
    g = torch.Generator().manual_seed(11)
    out, q = [], 0
    for i in range(n_batches):
        n = 2 + i % 3
        if kind == "videoqa":
            s = torch.randn(n, 5, generator=g)
            t = torch.randint(0, 5, (n, 1), generator=g)
            if i == no_gt_batch:
                t[:] = -1
        else:
            s = torch.randn(n, 1, generator=g) * 3
            t = torch.randint(0, 2, (n, 1), generator=g)
        out.append({"qids": list(range(q, q + n)), "targets": t, "s": s})
        q += n
    return out


def _qa_call(kind, batches):
    from hero_b200 import evalpass
    if kind == "videoqa":
        return evalpass.validate_videoqa(_ScoresOfBatch(), batches, "val", task="how2qa",
                                         save_logits=True)
    return evalpass.validate_violin(_ScoresOfBatch(), batches, "val", save_logits=True)


def _qa_case(rank, world, kind, n_batches, no_gt_batch):
    import time
    _Patch.setattr(time, "time", _StepClock())
    return _qa_call(kind, _qa_batches(kind, n_batches, no_gt_batch)[rank::world])


@pytest.mark.parametrize("kind", ["videoqa", "violin"])
@pytest.mark.parametrize("world, n_batches", [(2, 5), (3, 2)])
def test_validate_qa_merges_every_rank(monkeypatch, kind, world, n_batches):
    import time
    res = _run("_qa_case", world, kind, n_batches, None)
    monkeypatch.setattr(time, "time", _StepClock())
    want_log, want_results, want_logits = _qa_call(
        kind, _rank_order(_qa_batches(kind, n_batches), world))
    monkeypatch.undo()
    n_ex = sum(len(b["qids"]) for b in _qa_batches(kind, n_batches))
    assert len(want_results) == len(want_logits) == n_ex
    for val_log, results, logits in res:
        assert results == want_results and logits == want_logits
        rate = [k for k in val_log if k.endswith("ex_per_s")]
        # a 1 s wall time everywhere: the rate is the global example count on every rank
        assert len(rate) == 1 and val_log[rate[0]] == want_log[rate[0]] == n_ex
        fixed = {k: v for k, v in val_log.items() if k != rate[0]}
        assert fixed == {k: v for k, v in res[0][0].items() if k != rate[0]}
        _close(fixed, {k: v for k, v in want_log.items() if k != rate[0]})
        acc = [k for k in fixed if k.endswith("acc")]
        assert len(acc) == 1 and fixed[acc[0]] == want_log[acc[0]]


def test_videoqa_without_ground_truth_on_one_rank_logs_nothing_anywhere():
    res = _run("_qa_case", 2, "videoqa", 4, 3)           # batch 3: rank 1's second batch
    _, want_results, _ = _qa_call("videoqa", _rank_order(_qa_batches("videoqa", 4, 3), 2))
    for val_log, results, _ in res:
        assert val_log == {} and results == want_results


# ------------------------------------------------------------------ TVC decoding
def _tvc_batches():
    from hero_b200 import synth
    from tests.test_tvc_cpu import fixture
    c = json.loads(str(fixture()["config"]))
    return [synth.syn_tvc_batch(**dict(c["batch_args"], seed=21 + i), split="val")
            for i in range(2)]


def _tvc_call(tmp, batches):
    from hero_b200 import evalpass, synth
    from tests.test_tvc_cpu import _Stub, fixture, tvc_model
    tx = fixture()
    c = json.loads(str(tx["config"]))
    return evalpass.decode_tvc(tvc_model(tmp, tx), batches, max_step=c["max_step"],
                               bos=synth.BOS, eos=synth.EOS, tokenizer=_Stub())


def _tvc_case(rank, world):
    from tests import fake_tvc_ops
    fake_tvc_ops.install(_Patch)
    with tempfile.TemporaryDirectory() as tmp:
        return _tvc_call(Path(tmp), _tvc_batches()[rank::world])


@pytest.mark.parametrize("world", [2, 3])
def test_decode_tvc_gathers_every_rank(tmp_path, monkeypatch, world):
    from tests import fake_tvc_ops
    res = _run("_tvc_case", world)
    fake_tvc_ops.install(monkeypatch)
    want = _tvc_call(tmp_path, _rank_order(_tvc_batches(), world))
    assert len(want) == sum(len(b["clip_ids"]) for b in _tvc_batches())
    for got in res:
        assert got == want


# ------------------------------------------------------------------ corpus pass
H = 8


class _StubVideoEncoder(nn.Module):
    """v_encoder(batch, 'repr') = the batch's frames, zeroed at padded frames."""

    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(torch.zeros(1))
        self.config = SimpleNamespace(c_config=SimpleNamespace(hidden_size=H))

    def forward(self, batch, task):
        assert task == "repr"
        return batch["frames"] * batch["c_attn_masks"][..., None]


class _HostStager:
    def __init__(self, device, depth=3):
        pass

    def stage(self, hb):
        return (hb,), None, 0

    def release(self, slot, stream):
        pass


class _NoStream:
    def wait_event(self, event):
        pass


def _host_corpus_pass(patch):
    from hero_b200 import evalpass
    patch.setattr(evalpass, "BatchStager", _HostStager)
    patch.setattr(torch.cuda, "current_stream", lambda device=None: _NoStream())


def _clip_batches(lengths, rows):
    """One batch per entry: clips of the given lengths (padded to the longest) at the given
    corpus rows."""
    from hero_b200.plan import PLAN_KEY
    g = torch.Generator().manual_seed(5)
    out = []
    for lens in lengths:
        T = max(lens)
        mask = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None]).long()
        out.append({PLAN_KEY: "host", "c_attn_masks": mask,
                    "frames": torch.randn(len(lens), T, H, generator=g)})
    return out, [list(r) for r in rows]


# the longest clip (17 frames) is in batch 1: on rank 1
CLIPS = ([[3, 5], [17, 2, 4], [6], [9, 1]], [[6, 0], [3, 7, 1], [4], [2, 5]])


def _embed_case(rank, world, lengths, rows, n_videos):
    from hero_b200 import evalpass
    _host_corpus_pass(_Patch)
    batches, idx = _clip_batches(lengths, rows)
    try:
        return evalpass.embed_video_corpus(_StubVideoEncoder(), batches[rank::world], n_videos,
                                           max_clip_len=20, video_indices=idx[rank::world])
    except ValueError as e:
        return str(e)


@pytest.mark.parametrize("world, n_batches", [(2, 4), (3, 4), (3, 2)])
def test_embed_video_corpus_shards_clips_over_ranks(monkeypatch, world, n_batches):
    from hero_b200 import evalpass
    lengths, rows = CLIPS[0][:n_batches], CLIPS[1][:n_batches]
    n_videos = sum(len(r) for r in rows)
    if n_batches == 2:                       # rows 0..4: renumber the two batches' clips
        rows = [[3, 0], [1, 4, 2]]
    res = _run("_embed_case", world, lengths, rows, n_videos)
    _host_corpus_pass(monkeypatch)
    batches, idx = _clip_batches(lengths, rows)
    emb, masks = evalpass.embed_video_corpus(_StubVideoEncoder(), _rank_order(batches, world),
                                             n_videos, max_clip_len=20,
                                             video_indices=_rank_order(idx, world))
    assert emb.shape == (n_videos, 17, H) and masks.shape == (n_videos, 17)
    for got_emb, got_masks in res:
        assert torch.equal(got_emb, emb) and torch.equal(got_masks, masks)
        assert got_masks.dtype == masks.dtype


@pytest.mark.parametrize("rows, what", [([[0, 1], [1, 2], [3], [4, 5]], "more than once"),
                                        ([[0, 1], [2, 3], [4], [5, 7]], "by no rank: [6]"),
                                        ([[0, 1], [2, 3], [4], [5, 9]], "outside [0, 8): [9]")])
def test_embed_video_corpus_rejects_rows_not_claimed_once(rows, what):
    lengths = [[3, 5], [4, 2], [6], [9, 1]]
    res = _run("_embed_case", 2, lengths, rows, 8)
    for msg in res:
        assert isinstance(msg, str) and what in msg, msg


# ------------------------------------------------------------------ full-corpus retrieval
def _flow(kind, world, n_batches):
    """(batches, call): the query batches and the evaluation to run on them."""
    from hero_b200 import evalpass
    from tests.test_retrieval_cpu import _batches, _corpus, _golden, _StubQueryModel
    from tests.test_tvr_eval_cpu import _fixture, _flow_batches, _StubModel
    if kind.startswith("vcmr_eval"):
        fx, cfg, flow = _fixture()
        split = (9, 13) if n_batches == 2 else (5, 6, 4, 7)
        batches, rank_queries = _flow_batches(fx, cfg, flow["rows"], split)
        kw = dict(max_before_nms=cfg["max_before_nms"], max_after_nms=cfg["max_after_nms"],
                  nms_thd=cfg["nms_thd"], vfeat_interval=cfg["interval"])

        def call(bs, patch):
            gt = flow["ground_truth"]
            if kind == "vcmr_eval_own_gt":        # partial_query_data: this shard's queries only
                mine = {q for b in bs for q in b["qids"]}
                gt = [e for e in gt if e["desc_id"] in mine]
            patch.setattr(evalpass, "rank_queries", rank_queries)
            return evalpass.full_vcmr_eval(_StubModel(), SimpleNamespace(device="cpu"), bs,
                                           cfg["video_ids"], cfg["video2idx"], gt, **kw)
        return batches, call
    fx, cfg = _golden()
    split = (6, 4) if n_batches == 2 else (3, 2, 3, 2)
    batches, video_ids, video2idx = _batches(fx, split=split)
    if kind == "vr":
        def call(bs, patch):
            return evalpass.full_vr_predictions(_StubQueryModel(fx), _corpus(fx), bs, video_ids,
                                                video2idx, max_vr_video=cfg["K_VR"])
    else:
        def call(bs, patch):
            return evalpass.full_vcmr_predictions(
                _StubQueryModel(fx), _corpus(fx), bs, video_ids, video2idx,
                q2c_alpha=cfg["q2c_alpha"], max_vcmr_video=cfg["K"],
                min_pred_l=cfg["min_pred_l"], max_pred_l=cfg["max_pred_l"],
                max_before_nms=cfg["N"], vfeat_interval=1.5)
    return batches, call


def _install_rank_fakes(patch):
    from tests import fake_nms_ops, fake_rank_ops
    fake_rank_ops.install(patch)
    fake_nms_ops.install(patch)


def _retrieval_case(rank, world, kind, n_batches):
    _install_rank_fakes(_Patch)
    batches, call = _flow(kind, world, n_batches)
    return call(batches[rank::world], _Patch)


@pytest.mark.parametrize("kind", ["vcmr_eval", "vcmr_eval_own_gt", "vcmr_predictions", "vr"])
@pytest.mark.parametrize("world, n_batches", [(2, 4), (3, 4), (3, 2)])
def test_full_retrieval_evaluation_merges_every_rank(monkeypatch, kind, world, n_batches):
    res = _run("_retrieval_case", world, kind, n_batches)
    _install_rank_fakes(monkeypatch)
    batches, call = _flow(kind, world, n_batches)
    want = call(_rank_order(batches, world), monkeypatch)
    if kind.startswith("vcmr_eval"):
        assert list(want) == ["submission", "metrics", "submission_nms", "metrics_nms"]
    for got in res:
        assert list(got) == list(want)
        assert got == want
        assert json.dumps(got) == json.dumps(want)      # float reprs and key order too
