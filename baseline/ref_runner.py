"""Harness around the UNMODIFIED reference (staged in the git-ignored `oracle/_ref/` by
`oracle/stage_ref.py`, which `__graft_entry__.build()` runs) for bench.py's reference arms.
Nothing of hero_b200's model, kernels or engine is on this path: the reference's own `HierarchicalVlModel` (model/model.py:117-237) and
`CrossModalTrm` (model/encoder.py:297-352) run through stock PyTorch.

Un-vendored dependencies are replaced by in-memory stand-ins (SURVEY.md Appendix B):
  apex FusedLayerNorm -> torch.nn.LayerNorm (same semantics and parameter names);
  horovod.torch       -> a 1-rank identity shim, or (N > 1) a torch.distributed-backed shim of
                         the calls the path makes (`allreduce_` = mean over ranks, like Horovod's
                         default `average=True`, utils/distributed.py:38-39).

One "reference step" = what train_vcmr.py:202-239 does around the encoder on one batch:
`forward_repr` + `f_encoder(query, 'txt')` (model/pretrain.py:65-70), backward from fixed upstream
gradients, and at N > 1 the reference's own `all_reduce_and_rescale_tensors` (utils/distributed.py:
19-46) over the parameters' gradients.
"""
import itertools
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(os.path.dirname(HERE), "oracle", "_ref")


def available():
    return REF_DIR if os.path.isfile(os.path.join(REF_DIR, "model", "model.py")) else None


def install(dist_backed=False):
    """Registers the stand-in modules and puts oracle/_ref first on sys.path."""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    fln = mod("apex.normalization.fused_layer_norm", FusedLayerNorm=torch.nn.LayerNorm)
    mod("apex.normalization", fused_layer_norm=fln)
    mod("apex", normalization=sys.modules["apex.normalization"], amp=mod("apex.amp"))
    if dist_backed:
        import torch.distributed as dist

        def allreduce_(t, name=None, average=True):
            dist.all_reduce(t, op=dist.ReduceOp.AVG if average else dist.ReduceOp.SUM)
            return t

        def allgather(t, name=None):
            out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
            dist.all_gather(out, t.contiguous())
            return torch.cat(out, 0)

        hvd = mod("horovod.torch", size=dist.get_world_size, rank=dist.get_rank,
                  local_rank=lambda: int(os.environ.get("LOCAL_RANK", "0")),
                  local_size=dist.get_world_size, allreduce_=allreduce_, allgather=allgather,
                  allgather_async=allgather, synchronize=lambda h: h)
    else:
        hvd = mod("horovod.torch", size=lambda: 1, rank=lambda: 0, local_rank=lambda: 0,
                  local_size=lambda: 1, allgather=lambda t, name=None: t,
                  allreduce_=lambda t, name=None, average=True: t,
                  allgather_async=lambda t, name=None: t, synchronize=lambda h: h)
    mod("horovod", torch=hvd)
    mod("lmdb")
    mod("lz4")
    mod("lz4.frame", compress=None, decompress=None)
    mod("msgpack_numpy", patch=lambda: None)
    mod("toolz")
    mod("toolz.sandbox", unzip=lambda seq: zip(*seq))
    mod("cytoolz", concat=itertools.chain.from_iterable)
    mod("tensorboardX", SummaryWriter=object)
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)


def build_model(device, seed=0, train=True):
    """The reference's HierarchicalVlModel with its own config/hero_finetune.json (6 + 3 layers),
    random init through its own `initialize()` (model/model.py:338-345)."""
    from model.model import HierarchicalVlModel, VideoModelConfig
    torch.manual_seed(seed)
    cfg = VideoModelConfig(os.path.join(REF_DIR, "config", "hero_finetune.json"))
    model = HierarchicalVlModel(cfg, vfeat_dim=4352, max_frm_seq_len=100)
    if hasattr(model, "initialize"):
        model.initialize()
    model = model.to(device)
    return model.train() if train else model.eval()


def make_step(model, autocast_dtype=None, world=1, train=True):
    """Returns step(vb, qb, dclip, dq) -> clip_outputs."""
    device = next(model.parameters()).device
    params = [p for p in model.parameters()]
    if world > 1:
        from utils.distributed import all_reduce_and_rescale_tensors

    def step(vb, qb, dclip=None, dq=None):
        if train:
            for p in params:
                p.grad = None
        ctx = (torch.autocast(device.type, dtype=autocast_dtype) if autocast_dtype is not None
               else torch.autocast(device.type, enabled=False))
        with torch.set_grad_enabled(train), ctx:
            clip = model(vb, "repr")
            q = model.f_encoder(qb, "txt")[0]
        if train:
            torch.autograd.backward([clip, q], [dclip.to(clip.dtype), dq.to(q.dtype)])
            if world > 1:     # train_vcmr.py:236-239
                grads = [p.grad.data for p in params if p.requires_grad and p.grad is not None]
                all_reduce_and_rescale_tensors(grads, float(1))
        return clip

    return step
