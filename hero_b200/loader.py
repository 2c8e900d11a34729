"""Host -> device batch staging for the training loop.

`PrefetchLoader` keeps the reference's interface (data/loader.py:89-144: wrap a loader, iterate
device batches, transfers overlap compute on a side stream) with two changes that matter at
step times of a few milliseconds per 32-clip step with 112 MB of frame features per step:

* batches land in a small ring of preallocated device buffers (`BatchStager`) instead of fresh
  `.cuda()` allocations guarded by `record_stream`: cross-stream frees keep the caching allocator
  from recycling the 2 x 56 MB feature buffers in time, and every step then pays cudaMalloc
  (measured: 8 ms of host time per step);
* the packing plan (hero_b200.plan) is attached before the copy — built by the collate function,
  by a `PlanPool` of worker processes, or (fallback) in-process — and its index arrays are
  uploaded on the same side stream, so the forward pass never reads a mask back from the device.
"""
import collections

import torch

from .plan import PLAN_KEY, QA_PLAN_KEY, PlanPool, attach_plan, video_kind


class BatchStager:
    """Ring of `depth` device-resident copies of a batch (one or several dicts of tensors).

    stage(*host_dicts) copies into the next slot on the side stream and returns
    (device_dicts, ready_event, slot); the consumer makes its stream wait for `ready_event`, and
    calls release(slot) after enqueueing the work that reads the slot — the slot's next copy waits
    for that point. Buffers are (re)allocated only when a tensor's shape or dtype changes."""

    def __init__(self, device, depth=3):
        self.device = torch.device(device)
        self.depth = depth
        self.stream = torch.cuda.Stream(self.device)
        self._bufs = [dict() for _ in range(depth)]
        self._free = [None] * depth
        self._copied = [None] * depth
        self._n = 0

    def stage(self, *host_batches):
        slot = self._n % self.depth
        self._n += 1
        bufs = self._bufs[slot]
        out = []
        if self._copied[slot] is not None:
            # the host is about to rewrite this slot's pinned index buffers: its previous upload
            # (depth steps ago) must have left the host side
            self._copied[slot].synchronize()
        with torch.cuda.stream(self.stream):
            if self._free[slot] is not None:
                self.stream.wait_event(self._free[slot])
            for bi, hb in enumerate(host_batches):
                d = {}
                for k, v in hb.items():
                    if torch.is_tensor(v):
                        buf = bufs.get((bi, k))
                        if buf is None or buf.shape != v.shape or buf.dtype != v.dtype:
                            buf = torch.empty(v.shape, dtype=v.dtype, device=self.device)
                            bufs[(bi, k)] = buf
                        buf.copy_(v, non_blocking=True)
                        d[k] = buf
                    else:
                        d[k] = v
                plan = d.get(PLAN_KEY)
                if plan is not None:      # index arrays ride on the same stream, through the
                    plan.dev = None       # slot's own pinned + device buffers
                    plan.to(self.device, self._staging(bufs, (bi, "plan")))
                    joint = plan.__dict__.get("_joint")
                    if joint is not None:
                        joint.dev = None
                        joint.to(self.device, self._staging(bufs, (bi, "joint")))
                qplan = d.get(QA_PLAN_KEY)
                if qplan is not None:     # video QA / VIOLIN: the query-fused rows' plan likewise
                    qplan.dev = None
                    qplan.to(self.device, self._staging(bufs, (bi, "qa")))
                out.append(d)
            ready = torch.cuda.Event()
            ready.record(self.stream)
            self._copied[slot] = ready
        return out, ready, slot

    def _staging(self, bufs, key):
        def get(n):
            pair = bufs.get(key)
            if pair is None or pair[0].numel() < n:
                cap = 1 << max(int(n) - 1, 1).bit_length()
                pair = (torch.empty(cap, dtype=torch.int32, pin_memory=True),
                        torch.empty(cap, dtype=torch.int32, device=self.device))
                bufs[key] = pair
            return pair
        return get

    def release(self, slot, stream=None):
        ev = torch.cuda.Event()
        ev.record(stream if stream is not None else torch.cuda.current_stream(self.device))
        self._free[slot] = ev


def record_plans(batches, stream):
    """Plan index buffers that are allocator-managed (uploaded outside a BatchStager): tell the
    allocator that `stream` uses them (data/loader.py:135-138 does this for every tensor of the
    batch). Harmless for the stager's own long-lived buffers."""
    for b in batches:
        plan = b.get(PLAN_KEY)
        if plan is None:
            continue
        for p in (plan, plan.__dict__.get("_joint"), b.get(QA_PLAN_KEY)):
            if p is not None and p.dev is not None:
                p.dev.flat.record_stream(stream)


class PrefetchLoader:
    """data/loader.py:89-144 on a BatchStager. `loader` yields host batches: a dict (video batch,
    'repr' plan; a video_qa_collate batch gets the 'videoqa' plans, a violin_collate batch the
    'violin' ones) or a (video_dict, query_dict) pair for the fused `forward_repr_txt` path. Plans
    already attached by the collate function are used as they are; otherwise they are built two
    batches ahead in `plan_workers` processes (0: in this process)."""

    def __init__(self, loader, device=None, depth=3, plan_workers=0):
        self.loader = loader
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None \
            else torch.device(device)
        self.stager = BatchStager(self.device, depth)
        self.pool = PlanPool(plan_workers) if plan_workers > 0 else None

    def __len__(self):
        return len(self.loader)

    def _with_plans(self, it):
        """Host batches with plans attached, in order; pool results are requested two ahead."""
        pending = collections.deque()

        def pull():
            try:
                b = next(it)
            except StopIteration:
                return False
            pair = isinstance(b, (tuple, list))
            vb, qb = (dict(b[0]), dict(b[1])) if pair else (dict(b), None)
            need = vb.get(PLAN_KEY) is None
            fut = self.pool.submit(vb, qb) if (need and self.pool is not None) else None
            pending.append((vb, qb, pair, need, fut))
            return True

        for _ in range(2):
            pull()
        while pending:
            vb, qb, pair, need, fut = pending.popleft()
            pull()
            if fut is not None:
                PlanPool.attach(fut, vb, qb)
            elif need:
                attach_plan(vb, kind=video_kind(vb))
                if qb is not None:
                    attach_plan(qb, kind="txt")
            yield (vb, qb) if pair else vb

    def __iter__(self):
        cur = torch.cuda.current_stream(self.device)
        staged = None
        for hb in self._with_plans(iter(self.loader)):
            pair = isinstance(hb, tuple)
            nxt = self.stager.stage(*(hb if pair else (hb,))) + (pair,)
            if staged is not None:
                yield self._hand_over(staged, cur)
                # resumed: the consumer has enqueued its work on the batch just handed over
                self.stager.release(staged[2], cur)
            staged = nxt
        if staged is not None:
            yield self._hand_over(staged, cur)

    @staticmethod
    def _hand_over(staged, cur):
        batches, ready, _, pair = staged
        cur.wait_event(ready)
        record_plans(batches, cur)
        return tuple(batches) if pair else batches[0]

    def __getattr__(self, name):
        return getattr(self.loader, name)
