"""Data-parallel evaluation on the GPU over NCCL: `distributed.sum_over_ranks` and the merged
pretraining validation (evalpass._task_totals) on a one-rank NCCL group built inside the test, where
the merged result must be bitwise the one-process result with the same single device->host copy
per task and no added synchronisation; and, on a machine with two or more GPUs, a genuine two-rank
run against the one-process call (skipped otherwise).

sum_over_ranks runs under torch.cuda.set_sync_debug_mode("error"). The validation loop cannot: its
one copy per task is itself a synchronising call. There the sync debug mode is "warn", and the
merged run must report exactly as many synchronising calls as the run with no process group."""
import os
import socket
import warnings

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
DEV = "cuda"
RATES = ("tok_per_s", "feat_per_s", "ex_per_s")


@pytest.fixture
def one_rank_nccl(tmp_path):
    store = dist.FileStore(str(tmp_path / "store"), 1)
    dist.init_process_group("nccl", store=store, rank=0, world_size=1,
                            device_id=torch.device(DEV, 0))
    try:
        yield
    finally:
        dist.destroy_process_group()


def _sync_warnings(fn):
    """(fn(), number of synchronising CUDA calls torch reported while it ran)."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, sum("synchroniz" in str(w.message) for w in seen)


def test_sum_over_ranks_on_one_nccl_rank(one_rank_nccl):
    from hero_b200 import distributed as hd
    for dtype in (torch.float32, torch.float64):
        t = torch.randn(7, generator=torch.Generator().manual_seed(1)).to(DEV, dtype)
        hd.sum_over_ranks(t)                                   # warm-up (communicator)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = hd.sum_over_ranks(t)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert out.dtype == dtype and out.device == t.device
        assert torch.equal(out.view(torch.uint8), t.view(torch.uint8))


def _validate(tmp_path, model):
    from hero_b200 import evalpass
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import loaders
    ld = loaders(DEV, attach=True)
    copies = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(t, *a, **k):
        if t.is_cuda:
            copies.append(tuple(t.shape))
        return real_cpu(t, *a, **k)

    torch.Tensor.cpu = counting_cpu
    try:
        out, n_sync = _sync_warnings(lambda: evalpass.validate_pretrain(model, ld, pv.Opts))
    finally:
        torch.Tensor.cpu = real_cpu
    return {k: v for k, v in out.items() if not k.endswith(RATES)}, copies, n_sync


def test_merged_pretrain_validation_on_one_nccl_rank(tmp_path, monkeypatch):
    """No group / a one-rank group / the merge forced on that group: the same bits, one copy per
    task, and the merge (sum_over_ranks before the copy) adds no synchronisation."""
    from hero_b200 import evalpass
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model
    model = build_model(tmp_path, gu.load("pretrain_val_tiny.npz"), DEV)
    _validate(tmp_path, model)                                 # warm-up (library, caches)
    alone, copies, n_sync = _validate(tmp_path, model)
    assert len(copies) == len(pv.TASKS)
    dist.init_process_group("nccl", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0,
                            world_size=1, device_id=torch.device(DEV, 0))
    try:
        grouped, copies_g, n_sync_g = _validate(tmp_path, model)
        monkeypatch.setattr(evalpass, "_data_parallel", lambda: True)
        _validate(tmp_path, model)                             # warm-up of the merge
        merged, copies_m, n_sync_m = _validate(tmp_path, model)
    finally:
        dist.destroy_process_group()
    assert grouped == alone and merged == alone
    assert len(copies_g) == len(copies_m) == len(pv.TASKS)
    assert n_sync_g == n_sync_m == n_sync
    assert model.training


# ------------------------------------------------------------------ two ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _two_rank_worker(rank, world, port, tmp, ret):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    from pathlib import Path
    from hero_b200 import distributed as hd, evalpass
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model, loaders
    hd.init(backend="nccl")
    try:
        dev = f"cuda:{rank}"
        s = hd.sum_over_ranks(torch.tensor([0.25 * (rank + 1), 1.0], device=dev, dtype=torch.float64))
        model = build_model(Path(tmp) / str(rank), gu.load("pretrain_val_tiny.npz"), dev)
        ld = {t: bs[rank::world] for t, bs in loaders(dev, attach=True).items()}
        out = evalpass.validate_pretrain(model, ld, pv.Opts)
        ret[rank] = (s.cpu().tolist(), {k: v for k, v in out.items() if not k.endswith(RATES)})
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_pretrain_validation_matches_one_process(tmp_path):
    from hero_b200 import evalpass
    from tests import golden_util as gu
    from tests import pretrain_val_batches as pv
    from tests.test_pretrain_val_cpu import build_model, loaders
    for r in range(2):
        (tmp_path / str(r)).mkdir()
    ret = mp.Manager().dict()
    mp.spawn(_two_rank_worker, args=(2, _free_port(), str(tmp_path), ret), nprocs=2, join=True)
    model = build_model(tmp_path, gu.load("pretrain_val_tiny.npz"), DEV)
    ld = {t: [b for r in range(2) for b in bs[r::2]] for t, bs in loaders(DEV, True).items()}
    want = evalpass.validate_pretrain(model, ld, pv.Opts)
    negatives = ("vsm_valid/loss_overall", "vsm_valid/loss_neg_ctx", "vsm_valid/loss_neg_q")
    for r in range(2):
        s, got = ret[r]
        assert s == [0.75, 2.0]
        assert got == ret[0][1]
        for k, v in want.items():
            if k.endswith(RATES) or k in negatives:      # VSM negatives come from both ranks
                continue
            assert got[k] == pytest.approx(v, rel=1e-6, abs=1e-12), k
