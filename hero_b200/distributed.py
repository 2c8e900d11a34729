"""Data-parallel plumbing: the function names of the reference's utils/distributed.py on top of
torch.distributed (NCCL over NVLink / NVSwitch on a multi-GPU node, gloo in CPU tests) instead of
Horovod.

Semantics kept from the reference (SURVEY.md Appendix D.8):
  * `all_reduce_and_rescale_tensors(tensors, denom)`: Horovod's `allreduce_` AVERAGES, so the
    result is mean-over-ranks / denom (utils/distributed.py:19-46).
  * `broadcast_tensors(tensors, root)` (utils/distributed.py:103-151), `all_gather_list`,
    `any_broadcast` (utils/distributed.py:182-212).
  * `sum_over_ranks`: the evaluation merge of device sums (the reference sums host values from
    `all_gather_list`), in a fixed rank order so every rank holds the same bits.
  * `VsmAllgather`: forward all-gather, backward = own slice of the incoming gradient with no
    reduction (model/pretrain.py:427-447).
What changes is the mechanism: when the gradients already live in one flat buffer
(`FlatParams.ensure_flat_grads`) the exchange is ONE in-place `all_reduce(AVG)` on that buffer —
no pack / unpack copies; otherwise tensors are coalesced once. One process per GPU, launched by
torchrun-style environment variables.
"""
import os
import pickle
import sys

import torch
import torch.distributed as dist


def init(backend=None):
    """Join the job described by RANK / WORLD_SIZE / MASTER_ADDR / MASTER_PORT (torchrun).
    Returns (rank, world_size, local_rank); a no-op single-process job when unset."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
            dist.init_process_group(backend, rank=rank, world_size=world,
                                    device_id=torch.device("cuda", local_rank))
        else:
            dist.init_process_group(backend, rank=rank, world_size=world)
    return rank, world, local_rank


def size():
    return dist.get_world_size() if dist.is_initialized() else 1


def rank():
    return dist.get_rank() if dist.is_initialized() else 0


def _avg_inplace(buf):
    if size() == 1:
        return
    if dist.get_backend() == "nccl":
        dist.all_reduce(buf, op=dist.ReduceOp.AVG)     # ncclAvg: in-switch (NVLS) capable
    else:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM)
        buf.div_(size())


def all_reduce_flat(buf, rescale_denom=1.0):
    """Mean over ranks of a flat gradient buffer, in place."""
    _avg_inplace(buf)
    if rescale_denom != 1.0:
        buf.div_(rescale_denom)
    return buf


class FlatGradExchange:
    """The gradient exchange of `all_reduce_and_rescale_tensors` (utils/distributed.py:19-46) on the
    flat gradient buffer of a FlatParams: mean over ranks, in place, no pack / unpack.

    wire="bf16" (default): ranges are cast into a persistent bf16 staging buffer, all-reduced there
    and cast back — half the NVLink bytes of an fp32 exchange (the reference exchanged fp16
    gradients under apex O2, train_vcmr.py:234-239); every rank ends with bit-identical fp32
    values (they are the same bf16 numbers). wire="fp32": in-place ncclAllReduce(AVG).

    overlap=True: the flat buffer keeps the cross-modal embedding tables (41 % of the bytes, final
    only when backward ends) at the end of each parameter group (params.is_late_grad). Call
    `prepare()` before the forward of a step that will be exchanged: when the embedding backward —
    the last node of the graph — begins, the exchange of everything else is enqueued on a side
    stream and runs beside it; `all_reduce()` after backward then reduces only the embedding
    ranges and joins. Without `prepare()` (or if the graph differentiates the stacks in an unusual
    order) `all_reduce()` reduces the whole buffer, as before."""

    def __init__(self, flat, wire="bf16", overlap=True):
        assert wire in ("bf16", "fp32")
        self.flat, self.wire, self.overlap = flat, wire, overlap
        g = flat.ensure_flat_grads()
        self.stage = (torch.empty(g.numel(), dtype=torch.bfloat16, device=g.device)
                      if wire == "bf16" else None)
        self.comm_stream = torch.cuda.Stream(g.device) if (overlap and g.is_cuda) else None
        self._armed = False
        self._early_done = None
        self._n_fwd = self._n_bwd = 0

    def describe(self):
        how = ("stack / head gradients all-reduced on a side stream during the embedding "
               "backward, embedding tables after backward" if self.overlap and self.comm_stream
               else "one all-reduce of the flat gradient buffer after backward")
        return f"NCCL all-reduce(AVG), {self.wire} on the wire; {how}"

    # ---- reduction of flat ranges on the current stream ----------------------------------------
    def _reduce_ranges(self, g, ranges):
        for a, b in ranges:
            if b <= a:
                continue
            if self.stage is None:
                _avg_inplace(g[a:b])
            else:
                self.stage[a:b].copy_(g[a:b])
                _avg_inplace(self.stage[a:b])
                g[a:b].copy_(self.stage[a:b])

    # ---- hook protocol (functional.EXCHANGE_HOOK) ------------------------------------------------
    def prepare(self):
        """The gradients of the forward/backward that follows will be exchanged."""
        from . import functional
        self._armed = bool(self.overlap and self.comm_stream is not None and size() > 1)
        self._early_done = None
        self._n_fwd = self._n_bwd = 0
        functional.EXCHANGE_HOOK[0] = self if self._armed else None

    def stack_forward(self):
        self._n_fwd += 1

    def stack_backward(self):
        self._n_bwd += 1

    def embedding_backward_begins(self):
        if not self._armed or self._early_done is not None:
            return
        if self._n_fwd == 0 or self._n_bwd != self._n_fwd:
            return          # some stack is still to be differentiated: leave it to all_reduce()
        g = self.flat.grad_flat
        cur = torch.cuda.current_stream(g.device)
        ready = torch.cuda.Event()
        ready.record(cur)
        self.comm_stream.wait_event(ready)
        with torch.cuda.stream(self.comm_stream):
            self._reduce_ranges(g, self.flat.early_ranges())
            done = torch.cuda.Event()
            done.record(self.comm_stream)
        self._early_done = done

    def all_reduce(self, rescale_denom=1.0):
        from . import functional
        g = self.flat.ensure_flat_grads()
        if size() > 1:
            if self._early_done is not None:
                self._reduce_ranges(g, self.flat.late_ranges())
                torch.cuda.current_stream(g.device).wait_event(self._early_done)
            else:
                self._reduce_ranges(g, [(0, g.numel())])
        self._early_done = None
        self._armed = False
        functional.EXCHANGE_HOOK[0] = None
        if rescale_denom != 1.0:
            g.div_(rescale_denom)
        return g

    def ranks_agree(self):
        """True iff every rank holds a bit-identical gradient buffer (collective call)."""
        g = self.flat.ensure_flat_grads()
        bits = g.view(torch.int32).to(torch.int64)
        digest = torch.stack([bits.sum(), (bits * (torch.arange(bits.numel(), device=g.device) % 8191
                                                   + 1)).sum()])
        if size() == 1:
            return True
        all_d = [torch.empty_like(digest) for _ in range(size())]
        dist.all_gather(all_d, digest)
        return all(bool((d == all_d[0]).all()) for d in all_d)

    def self_check(self):
        """Known-answer test of the exchange on this job's ranks and transport: rank r fills the
        buffer with (r + 1) * base, base a fixed pattern of multiples of 1/16 (exact in bf16);
        afterwards every rank must hold base * (W + 1) / 2 and all ranks must hold bit-identical
        buffers. With the bf16 wire the partial sums of W > 4 ranks are no longer all exact in
        bf16 (e.g. 21 * 13/16): the bound is one rounding (2^-9 relative) per addition plus the
        final one. Leaves the buffer zeroed."""
        g = self.flat.ensure_flat_grads()
        W, r = size(), rank()
        base = ((torch.arange(g.numel(), device=g.device) % 31) - 15).float() / 16.0
        g.copy_(base * (r + 1))
        self.all_reduce()
        want = base * ((W + 1) / 2.0)
        tol = (max(2.0 ** -7, (W + 1) * 2.0 ** -9) if self.stage is not None else 2.0 ** -20)
        err = float(((g - want).abs() - tol * want.abs()).max().item())
        same = self.ranks_agree()
        g.zero_()
        if err > 1e-6 or not same:
            raise RuntimeError(f"gradient all-reduce self-check failed on rank {r}: max excess "
                               f"error {err:.3e}, ranks bit-identical: {same}")
        return f"ok (mean of rank patterns reproduced on {W} ranks, bit-identical across ranks)"


def all_reduce_and_rescale_tensors(tensors, rescale_denom):
    """utils/distributed.py:19-46. Tensors that are consecutive views of one storage are reduced
    in place as a single message; anything else is coalesced once."""
    tensors = list(tensors)
    if not tensors:
        return
    flat = _as_single_view(tensors)
    if flat is not None:
        all_reduce_flat(flat, float(rescale_denom))
        return
    buf = torch.cat([t.reshape(-1) for t in tensors])
    all_reduce_flat(buf, float(rescale_denom))
    off = 0
    for t in tensors:
        n = t.numel()
        t.view(-1).copy_(buf[off:off + n])
        off += n


def _as_single_view(tensors):
    """If the tensors tile one contiguous region of a single storage (gaps allowed only as the
    alignment padding of FlatParams, which holds zeros), return that region as one tensor."""
    t0 = tensors[0]
    if not all(t.is_contiguous() and t.dtype == t0.dtype and t.device == t0.device and
               t.untyped_storage().data_ptr() == t0.untyped_storage().data_ptr()
               for t in tensors):
        return None
    es = t0.element_size()
    lo = min(t.data_ptr() for t in tensors)
    hi = max(t.data_ptr() + t.numel() * es for t in tensors)
    covered = sum(t.numel() for t in tensors)
    total = (hi - lo) // es
    if total > covered + 64 * len(tensors):     # more than alignment slack: not one region
        return None
    base = t0.untyped_storage().data_ptr()
    out = torch.empty(0, dtype=t0.dtype, device=t0.device)
    out.set_(t0.untyped_storage(), (lo - base) // es, (total,), (1,))
    return out


def broadcast_tensors(tensors, root_rank, buffer_size=None):
    """utils/distributed.py:103-151: every rank ends with root's values."""
    if size() == 1:
        return
    tensors = list(tensors)
    flat = _as_single_view(tensors) if tensors else None
    if flat is not None:
        dist.broadcast(flat, root_rank)
        return
    for t in tensors:
        dist.broadcast(t, root_rank)


def all_gather_list(data):
    """utils/distributed.py:182-198: gather arbitrary picklable data from all ranks. Stays off the
    GPU critical path (object collectives), unlike the reference's byte-tensor + .item() version."""
    if size() == 1:
        return [pickle.loads(pickle.dumps(data))]
    out = [None] * size()
    dist.all_gather_object(out, data)
    return out


def sum_over_ranks(t):
    """Sum over ranks of a small fp32 / fp64 tensor (metric sums and counts), on its device and
    without a host synchronisation: one all_gather_into_tensor into a (W, n) buffer, then the rows
    added in rank order. The order of the additions is fixed, so the result is bitwise the same on
    every rank; all_reduce(SUM) would leave it to NCCL's algorithm. Returns a new tensor of t's
    shape (a copy of t without a process group). Host data goes through `all_gather_list`."""
    if t.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"sum_over_ranks takes fp32 / fp64 tensors, not {t.dtype}")
    flat = t.detach().reshape(-1).contiguous()
    if not dist.is_initialized():
        return flat.clone().view(t.shape)
    world = dist.get_world_size()
    rows = torch.empty(world * flat.numel(), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(rows, flat)
    rows = rows.view(world, flat.numel())
    out = rows[0].clone()
    for r in range(1, world):
        out += rows[r]
    return out.view(t.shape)


def any_broadcast(data, root_rank):
    """utils/distributed.py:201-212."""
    if size() == 1:
        return pickle.loads(pickle.dumps(data))
    box = [data if rank() == root_rank else None]
    dist.broadcast_object_list(box, src=root_rank)
    return box[0]


def bucket_parts(a, b, world, align=64):
    """Split the flat range [a, b) into `world` consecutive parts of `chunk` elements (a multiple of
    `align`; the last parts may be short or empty). Returns (parts, chunk)."""
    n = b - a
    chunk = (-(-n // world) + align - 1) // align * align
    parts = [(min(a + r * chunk, b), min(a + (r + 1) * chunk, b)) for r in range(world)]
    return parts, chunk


class PeerExchange:
    """Mean all-reduce of ranges of the flat gradient buffer with DMA copies over NVLink instead of
    a communication kernel (the buckets that travel while backward is still running).

    The gradient buffer and a staging buffer live in symmetric memory
    (torch.distributed._symmetric_memory: every rank maps every peer's allocation). For a bucket
    [a, b) split into `world` parts, rank r owns part r:
      1. reduce-scatter: every rank copies its values of part r into a staging slot on rank r
         (cudaMemcpyAsync to the peer mapping = copy engines, no SMs) and signals r;
      2. rank r adds the world-1 slots to its own values and scales by 1/world
         (`hero_reduce_slots_f32`, the only kernel: <= 16 CTAs, HBM-bound);
      3. all-gather: rank r copies the reduced part into every peer's gradient buffer and signals.
    Everything is enqueued on one side stream, ordered after the event that marks the bucket
    final. NCCL kernels cannot do this job beside the GEMMs: the GEMMs run one CTA per SM, a
    full-speed NCCL kernel wants ~24 SMs, a 4-8 CTA one moves 90-170 GB/s and was measured to finish
    only after backward (tools/dp_timeline.py, tools/allreduce_probe.py)."""

    def __init__(self, flat, group=None):
        import torch.distributed._symmetric_memory as symm
        group = dist.group.WORLD if group is None else group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        dev = flat.flat.device
        try:
            symm.enable_symm_mem_for_group(group.group_name)
        except Exception:       # newer torch enables every group implicitly
            pass
        pad = 64 * self.world
        self.grad = symm.empty(flat.total + pad, dtype=torch.float32, device=dev)
        self.stage = symm.empty(flat.total + pad, dtype=torch.float32, device=dev)
        self.h_grad = symm.rendezvous(self.grad, group.group_name)
        self.h_stage = symm.rendezvous(self.stage, group.group_name)
        self.grad.zero_()
        self.stream = torch.cuda.Stream(dev, priority=-1)
        self.channels = max(1, min(128, self.h_grad.signal_pad_size // (4 * self.world) - 1))
        self.flat = flat
        flat.adopt_grad_buffer(self.grad)
        torch.cuda.synchronize(dev)
        self.h_grad.barrier(0)

    def fits(self, a, b):
        _, chunk = bucket_parts(a, b, self.world)
        return (self.world - 1) * chunk <= b - a      # staging of a bucket stays inside [a, b)

    def exchange(self, a, b, event=None, reduce_ctas=16):
        """Enqueue the exchange of [a, b) behind `event` (default: behind everything already on
        the current stream). `reduce_ctas` caps the reduction kernel (small beside backward)."""
        if event is None:
            event = torch.cuda.Event()
            event.record()
        self.stream.wait_event(event)
        with torch.cuda.stream(self.stream):
            self._scatter(a, b)
            self._reduce(a, b, reduce_ctas)
            self._gather(a, b)

    def _others(self):
        return [(self.rank + k) % self.world for k in range(1, self.world)]

    def _plan(self, a, b):
        """Views and peer mappings of a bucket (the same buckets recur every step: cached)."""
        plans = self.__dict__.setdefault("_plans", {})
        pl = plans.get((a, b))
        if pl is None:
            W, me = self.world, self.rank
            parts, chunk = bucket_parts(a, b, W)
            lo, hi = parts[me]
            # one signal channel per bucket (pads hold >= 128 channels): a bucket's signals never
            # queue behind another bucket's, and the "gathered" acknowledgements can all be
            # collected at the end of the step instead of stalling the stream after every bucket
            pl = {"chunk": chunk, "lo": lo, "hi": hi, "scatter": [], "gather": [],
                  "channel": len(plans) % self.channels,
                  "wait_gather": [p for p in self._others() if parts[p][1] > parts[p][0]]}
            for r in self._others():
                rlo, rhi = parts[r]
                if rhi > rlo:
                    slot = (me - r - 1) % W        # 0 .. W-2: which of r's slots is mine
                    dst = self.h_stage.get_buffer(r, (rhi - rlo,), torch.float32,
                                                  a + slot * chunk)
                    pl["scatter"].append((r, dst, self.grad[rlo:rhi]))
                if hi > lo:
                    dst = self.h_grad.get_buffer(r, (hi - lo,), torch.float32, lo)
                    pl["gather"].append((r, dst))
            if hi > lo:
                assert (hi - lo) % 4 == 0 and lo % 4 == 0   # FlatParams aligns everything to 64
                pl["mine"] = self.grad[lo:hi]
                pl["slots"] = self.stage[a:]
            plans[(a, b)] = pl
        return pl

    def _scatter(self, a, b):
        """1. my values of part r -> r's staging slot for me, then tell r."""
        pl = self._plan(a, b)
        for r, dst, src in pl["scatter"]:
            dst.copy_(src, non_blocking=True)
            self.h_stage.put_signal(r, pl["channel"])

    def _reduce(self, a, b, reduce_ctas=16):
        """2. once every peer's slice of my part has arrived: mean into my gradients."""
        from . import ops
        pl = self._plan(a, b)
        if pl["hi"] > pl["lo"]:
            for p in self._others():
                self.h_stage.wait_signal(p, pl["channel"])
            ops.reduce_slots(pl["mine"], pl["slots"], self.world - 1, pl["chunk"],
                             1.0 / self.world, max_ctas=reduce_ctas)

    def _gather(self, a, b):
        """3. my reduced part -> every peer's gradient buffer; wait for theirs."""
        pl = self._plan(a, b)
        for r, dst in pl["gather"]:
            dst.copy_(pl["mine"], non_blocking=True)
            self.h_grad.put_signal(r, pl["channel"])
        self.__dict__.setdefault("_unacked", []).append(pl)

    def join(self):
        """Collect the peers' "gathered" signals of every bucket of the step, then make the current
        stream wait for every exchange enqueued so far."""
        with torch.cuda.stream(self.stream):
            for pl in self.__dict__.pop("_unacked", []):
                for p in pl["wait_gather"]:
                    self.h_grad.wait_signal(p, pl["channel"])
        ev = torch.cuda.Event()
        ev.record(self.stream)
        torch.cuda.current_stream().wait_event(ev)


class GradBucketer:
    """Overlaps the data-parallel gradient exchange with the rest of the backward pass.

    The reference all-reduces one flat copy of every gradient AFTER backward has finished
    (utils/distributed.py:19-46, called at train_vcmr.py:233-239). Here gradients are accumulated
    in place in FlatParams' flat fp32 buffer, and the hand-written transformer backward reports
    each layer's parameters as soon as their gradient is final: the ranges of the flat buffer they
    cover are all-reduced (mean) right away on the communicator's stream while the layers below
    are still being differentiated. `finish()` reduces every range not covered so far and waits.
    The result equals one all_reduce_flat(grad_flat) after backward.

    Usage (one step):
        with bucketer:                 # installs the hook for forward + backward
            loss = model(...); loss.backward()
        bucketer.finish(); optimizer.step()

    A parameter used by several forward calls (e.g. c_encoder for video rows and again for query
    rows) is exchanged only after its LAST backward: forward registers every use (`expect`),
    backward retires them (`ready`)."""

    def __init__(self, flat, min_elems=1 << 20, overlap_ctas=0, transport="auto"):
        """transport: how buckets travel while backward is running —
        "p2p" (PeerExchange: symmetric memory + copy engines, NCCL backend only), "nccl"
        (an extra communicator capped at `overlap_ctas` CTAs, with the compute kernels sized for
        that many fewer SMs), "auto" = p2p when available else the default communicator.
        The remainder after backward always goes through the default, full-speed communicator."""
        self.flat = flat
        self.min_elems = min_elems       # merge announced ranges into messages of >= 4 MB
        self.overlap_ctas = overlap_ctas
        self.pg = None
        self.p2p = None
        self.p2p_tail_max_world = 0
        nccl = size() > 1 and dist.get_backend() == "nccl"
        if nccl and transport in ("auto", "p2p"):
            try:
                self.p2p = PeerExchange(flat)
            except Exception as e:          # no symmetric memory on this system
                if transport == "p2p":
                    raise
                import warnings
                warnings.warn(f"GradBucketer: peer exchange unavailable ({e!r}); using NCCL")
        if nccl and self.p2p is None and overlap_ctas > 0:
            opts = dist.ProcessGroupNCCL.Options()
            opts.config.max_ctas = overlap_ctas
            opts.config.min_ctas = 1
            # its CTAs must win the SMs the compute kernels leave free as soon as they are free:
            # without priority the exchange kernel sat behind the thousands of queued attention /
            # LayerNorm CTAs and only ran after backward had finished (tools/dp_timeline.py)
            opts.is_high_priority_stream = True
            self.pg = dist.new_group(backend="nccl", pg_options=opts)
        self.reset()

    def reset(self):
        self.pending = {}       # id(param) -> forward uses whose backward has not run yet
        self.done = []          # [a, b) ranges of the flat buffer already handed to the backend
        self.handles = []
        self.queue = []         # final but not yet sent ranges (waiting to reach min_elems)

    # ---- hook protocol (hero_b200.functional.GRAD_HOOK) -------------------------------------
    def expect(self, params):
        for p in params:
            self.pending[id(p)] = self.pending.get(id(p), 0) + 1

    wants_events = True      # the stack backward stays one native call (functional.py)

    def ready(self, params, event=None):
        """`event`: CUDA event after which the gradients of `params` are complete (else: complete
        in current-stream order at the time of the call)."""
        gf = self.flat.grad_flat
        if gf is None or size() == 1:
            return
        base, spans = gf.data_ptr(), []
        for p in params:
            k = id(p)
            left = self.pending.get(k, 1) - 1
            self.pending[k] = left
            ent = self.flat._by_id.get(k)
            if left > 0 or ent is None or p.grad is None:
                continue
            if p.grad.data_ptr() != base + 4 * ent[0]:
                continue                # gradient does not live in the flat buffer: finish() only
            spans.append(ent)
        for off, n in sorted(spans):
            end = min((off + n + 63) // 64 * 64, self.flat.total)   # alignment padding is zeros
            if self.queue and off <= self.queue[-1][1]:
                self.queue[-1][1] = max(self.queue[-1][1], end)
            else:
                self.queue.append([off, end])
        if sum(b - a for a, b in self.queue) >= self.min_elems:
            self._flush(event)

    def __enter__(self):
        from . import functional, ops
        self.reset()
        functional.GRAD_HOOK[0] = self
        if self.pg is not None:
            ops.set_sm_limit(0)
            ops.set_sm_limit(max(ops.sm_count() - self.overlap_ctas, 1))
        return self

    def __exit__(self, *exc):
        from . import functional, ops
        functional.GRAD_HOOK[0] = None
        if self.pg is not None:
            ops.set_sm_limit(0)
        return False

    # ---- exchange ------------------------------------------------------------------------------
    def _launch(self, a, b, group=None):
        if b <= a:
            return
        buf = self.flat.grad_flat[a:b]
        if dist.get_backend() == "nccl":
            self.handles.append((dist.all_reduce(buf, op=dist.ReduceOp.AVG, group=group,
                                                 async_op=True), None))
        else:
            self.handles.append((dist.all_reduce(buf, op=dist.ReduceOp.SUM, async_op=True), buf))
        self.done.append((a, b))

    def _flush(self, event=None):
        for a, b in self.queue:
            if self.p2p is not None and self.p2p.fits(a, b):
                self.p2p.exchange(a, b, event)   # beside the backward: copy engines
                self.done.append((a, b))
            else:
                if event is not None:            # NCCL orders itself after the current stream
                    torch.cuda.current_stream().wait_event(event)
                self._launch(a, b, self.pg)      # (capped) communicator
        self.queue = []

    def finish(self, rescale_denom=1.0):
        """Exchange every range not sent so far, wait for all of it (the current stream waits; the
        host does not block on NCCL) and apply the reference's rescale."""
        timing = os.environ.get("HERO_DP_TIMING") == "1"
        marks = []

        def mark(name):
            if timing:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((name, e))

        if size() > 1:
            self.flat.ensure_flat_grads()
            mark("backward enqueued work done")
            rest = [tuple(r) for r in self.queue]
            self.queue = []
            pos = 0
            for a, b in sorted(self.done):
                if a > pos:
                    rest.append((pos, a))
                pos = max(pos, b)
            if pos < self.flat.total:
                rest.append((pos, self.flat.total))
            # After backward nothing competes for SMs: the remainder goes through the full-speed
            # NCCL communicator (176 MB in 0.5-0.6 ms at N = 2; the peer-copy path was measured at
            # 0.7-0.8 ms for the same bytes - `p2p_tail_max_world` > 0 re-enables it for A/B runs).
            for a, b in rest:
                if self.p2p is not None and size() <= self.p2p_tail_max_world and self.p2p.fits(a, b):
                    self.p2p.exchange(a, b, reduce_ctas=592)
                else:
                    self._launch(a, b)
            n_tail = len(self.handles)
            for h, buf in self.handles:
                h.wait()
                if buf is not None:
                    buf.div_(size())
            mark(f"remainder through NCCL ({n_tail} calls)")
            if self.p2p is not None:
                self.p2p.join()
                mark("peer exchanges joined")
        if rescale_denom != 1.0:
            self.flat.grad_flat.div_(rescale_denom)
        if timing and marks:
            torch.cuda.synchronize()
            print("GradBucketer.finish device ms:",
                  [(b[0], round(a[1].elapsed_time(b[1]), 3)) for a, b in zip(marks[:-1], marks[1:])],
                  file=sys.stderr)
        self.reset()


def overlapped_exchange(flat, transport="none", **kw):
    """The gradient-exchange schedule for a training loop: None = one NCCL all-reduce of the flat
    buffer after backward (`all_reduce_flat`, the reference's schedule — the default), or a
    GradBucketer ("p2p": buckets travel as peer copies during backward, "nccl": through a capped
    communicator).

    The bucketer pays ~100 extra host-side enqueues per step and 2 (N-1) copies and signals per
    bucket per rank, and the 41 % of the bytes that become final only when backward ends stay
    exposed either way, so it is opt-in (not measured on H100)."""
    if size() <= 1 or transport in (None, "none"):
        return None
    return GradBucketer(flat, transport=transport, **kw)


class VsmAllgather(torch.autograd.Function):
    """model/pretrain.py:427-447: all-gather along dim 0 in rank order (ranks may contribute
    different row counts, as hvd.allgather allows); the backward hands each rank the slice of the
    gradient that corresponds to its own rows (no reduction)."""

    @staticmethod
    def forward(ctx, tensor, name=None, equal_counts=False):
        ctx.span = (0, tensor.shape[0])
        if size() == 1:
            return tensor
        tensor = tensor.contiguous()
        if equal_counts:
            # every rank contributes tensor.shape[0] rows (stated by the caller): one collective
            # into a preallocated block, nothing read back to the host
            n0 = tensor.shape[0]
            out = torch.empty((n0 * size(),) + tuple(tensor.shape[1:]), dtype=tensor.dtype,
                              device=tensor.device)
            dist.all_gather_into_tensor(out, tensor)
            ctx.span = (rank() * n0, (rank() + 1) * n0)
            return out
        n = torch.tensor([tensor.shape[0]], dtype=torch.int64, device=tensor.device)
        counts = [torch.zeros_like(n) for _ in range(size())]
        dist.all_gather(counts, n)
        counts = [int(c.item()) for c in counts]
        rest = tuple(tensor.shape[1:])
        if len(set(counts)) == 1:
            out = torch.empty((sum(counts),) + rest, dtype=tensor.dtype, device=tensor.device)
            dist.all_gather_into_tensor(out, tensor)
        else:
            mx = max(counts)
            padded = tensor.new_zeros((mx,) + rest)
            padded[:tensor.shape[0]] = tensor
            parts = [torch.empty_like(padded) for _ in range(size())]
            dist.all_gather(parts, padded)
            out = torch.cat([p[:c] for p, c in zip(parts, counts)], 0)
        start = sum(counts[:rank()])
        ctx.span = (start, start + counts[rank()])
        return out

    @staticmethod
    def backward(ctx, grad_output):
        a, b = ctx.span
        return grad_output[a:b], None, None


vsm_allgather = VsmAllgather.apply
