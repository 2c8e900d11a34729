"""Forward-only passes and checkpoint I/O around the encoder (SURVEY.md §8f rank 4).

* `embed_video_corpus` — the video-embedding pass of eval_vcmr.py:161-203: every clip of a corpus
  through `v_encoder(batch, 'repr')` in eval mode, results scattered into one
  (n_videos, max_clip_len, H) tensor + mask, batch by batch. Here the batches are staged through a
  `loader.BatchStager` ring (next batch's H2D copy and plan upload overlap the current forward) and
  the packed encoder runs without an autograd graph (activations ping-pong between two workspace
  slots, `hero_bert_stack_fwd` with save=False).
* `VideoCorpus` / `rank_queries` / `full_vcmr_predictions` / `full_vr_predictions` — the ranking
  half of eval_vcmr.py:205-418 and eval_vr.py:198-260: video scores, span probabilities and
  moment lists of every query against the whole corpus, on the kernels of csrc/rank.cu (DESIGN §4
  "Retrieval ranking"). No (Nq, K, L, L) tensor, no full sort, one small device->host copy per
  query batch.
* `nms_moments` / `eval_retrieval` / `full_vcmr_eval` — the rest of eval_vcmr.py:205-508:
  temporal NMS of the ranked lists on the device (csrc/nms.cu), carried home in the same copy, and
  the TVR recall metrics of utils/tvr_standalone_eval.py vectorised over queries on the host
  (DESIGN §4 "Temporal NMS and TVR metrics").
* `validate_videoqa` — eval_videoQA.py:120-173 on HeroForVideoQA.
* `validate_violin` — eval_violin.py:118-164 on HeroForViolin.
* `validate_pretrain` (and `validate_mlm` / `_mffr` / `_mfm_nce` / `_fom` / `_vsm`) —
  pretrain.py:387-608: the fused LM-head GEMM with `hero_ce_finish_stats` for MLM and MFM-NCE (no
  logits tensor), `hero_row_l2_cos` for l2 / cosine, sums on the device, one device->host copy per
  task (DESIGN §4 "Pretraining validation").
* `decode_tvc` — TVC captions of inf_tvc.py / train_tvc.py: greedy (the reference's), beam
  search or sampling, with optional n-gram blocking and minimum length.
* `ModelSaver` / `TrainingRestorer` — utils/save.py:112-181 with the same file layout (`vocab_padded`
  flag, `model_step_<n>.pt`, `train_state_<n>.pt`, `restore.pt` + backup), so checkpoints are
  interchangeable with the reference's; optimizer state is FusedAdamW's flat moments.

Data-parallel evaluation (DESIGN §4 "Data-parallel evaluation"): when `distributed.size() > 1`,
every evaluation entry point above evaluates what its own rank was given (its loader's batches,
its corpus clips, its query batches and their ground truth) and returns the result merged over all
ranks, the same on every rank. Device sums go through `distributed.sum_over_ranks`, host records
and dicts through `distributed.all_gather_list`. Without a process group, or with one rank,
nothing is exchanged.
"""
import os
from collections import OrderedDict
from os.path import exists, join

import numpy as np
import torch

from . import distributed, ops
from .loader import BatchStager
from .plan import PLAN_KEY, attach_plan


def _data_parallel():
    """True when the evaluation is sharded: each rank evaluates the batches it was given and every
    entry point returns the result merged over all ranks."""
    return distributed.size() > 1


@torch.no_grad()
def embed_video_corpus(model, batches, n_videos, max_clip_len, device=None, video_indices=None,
                       out_dtype=torch.float32):
    """`batches`: iterable of HOST video batch dicts (reference `video_collate` layout; plans are
    attached here when the collate has not). `video_indices`: per batch the row of each clip in the
    corpus tensors (default: consecutive). Returns (frame_embeddings (n_videos, max_clip_len', H),
    c_attn_masks (n_videos, max_clip_len')) trimmed to the longest clip seen, like the reference.

    Data-parallel (`distributed.size() > 1`), each rank embeds the clips of its own `batches` at
    their global rows, and every rank returns the whole corpus: the rows of all ranks must cover
    0..n_videos-1 exactly once (checked on the gathered host indices before any collective,
    ValueError otherwise), the trim is to the longest clip of any rank, and the zero-initialised
    corpus and masks are summed over ranks (each row has one writer, so the sum is exact). A rank
    without clips still joins; its corpus is allocated with the model's hidden size."""
    v_enc = model.v_encoder if hasattr(model, "v_encoder") else model
    device = device or next(v_enc.parameters()).device
    was_training = v_enc.training
    v_enc.eval()
    stager = BatchStager(device, depth=3)
    cur = torch.cuda.current_stream(device)
    total, masks, longest, row = None, None, 0, 0
    sharded = _data_parallel()
    claimed = []                                         # host rows of this rank's clips
    it = iter(batches)

    def stage_next():
        try:
            hb = dict(next(it))
        except StopIteration:
            return None
        if hb.get(PLAN_KEY) is None:
            attach_plan(hb)
        return stager.stage(hb)

    nxt = stage_next()
    bi = 0
    while nxt is not None:
        (batch,), ready, slot = nxt
        cur.wait_event(ready)
        emb = v_enc(batch, "repr")                       # (B, T, H), zeros at padded frames
        stager.release(slot, cur)
        nxt = stage_next()                               # next copy overlaps this forward
        B, T, Hd = emb.shape
        assert T <= max_clip_len, f"clip of {T} frames exceeds max_clip_len {max_clip_len}"
        if total is None:
            total = torch.zeros((n_videos, max_clip_len, Hd), dtype=out_dtype, device=device)
            masks = torch.zeros((n_videos, max_clip_len), dtype=batch["c_attn_masks"].dtype,
                                device=device)
        if sharded:
            rows = (np.asarray(video_indices[bi], dtype=np.int64).reshape(-1)
                    if video_indices is not None else np.arange(row, row + B))
            claimed.append(rows)
            if rows.size and (rows.min() < 0 or rows.max() >= n_videos):
                rows = None             # reported by every rank in _merge_corpus, not written
        if video_indices is not None:
            idx = torch.as_tensor(video_indices[bi], device=device, dtype=torch.long)
        else:
            idx = torch.arange(row, row + B, device=device)
        if not sharded or rows is not None:
            total[idx, :T] = emb.to(out_dtype)
            masks[idx, :T] = batch["c_attn_masks"]
        longest = max(longest, T)
        row += B
        bi += 1
    if was_training:
        v_enc.train()
    if sharded:
        return _merge_corpus(v_enc, total, masks, longest, claimed, n_videos, max_clip_len,
                             device, out_dtype)
    if total is None:
        return None, None
    return total[:, :longest], masks[:, :longest]


def _merge_corpus(v_enc, total, masks, longest, claimed, n_videos, max_clip_len, device,
                  out_dtype):
    """The data-parallel end of `embed_video_corpus`: one host gather of every rank's rows,
    longest clip and mask dtype; the row check; then the corpus and masks all-reduced (SUM) and
    trimmed to the longest clip of any rank."""
    import torch.distributed as dist
    mine = np.concatenate(claimed) if claimed else np.zeros(0, dtype=np.int64)
    parts = distributed.all_gather_list((mine, longest, None if masks is None else masks.dtype))
    rows = np.concatenate([p[0] for p in parts])
    inside = rows[(rows >= 0) & (rows < n_videos)]
    count = np.bincount(inside, minlength=n_videos)
    outside = np.setdiff1d(rows, inside)
    twice, missing = np.flatnonzero(count > 1), np.flatnonzero(count == 0)
    if len(outside) or len(twice) or len(missing):
        raise ValueError(
            f"data-parallel corpus of {n_videos} clips: every row must be embedded by exactly one "
            f"rank; rows outside [0, {n_videos}): {outside[:8].tolist()}, claimed more than once: "
            f"{twice[:8].tolist()}, claimed by no rank: {missing[:8].tolist()} (first 8 of each)")
    longest = max(p[1] for p in parts)
    if longest == 0:
        return None, None
    if total is None:
        mask_dtype = next(p[2] for p in parts if p[2] is not None)
        hidden = v_enc.config.c_config.hidden_size
        total = torch.zeros((n_videos, max_clip_len, hidden), dtype=out_dtype, device=device)
        masks = torch.zeros((n_videos, max_clip_len), dtype=mask_dtype, device=device)
    # the full buffers, not contiguous copies of the trimmed ones: no second corpus in memory
    dist.all_reduce(total, op=dist.ReduceOp.SUM)
    dist.all_reduce(masks, op=dist.ReduceOp.SUM)
    return total[:, :longest], masks[:, :longest]


# ------------------------------------------------------------------ full-corpus ranking
RANK_TASKS = ("VR", "VCMR", "SVMR")
MAX_SELECT = 1024          # top-K clips and top-N moments per query (csrc/rank.cu)
MAX_CLIP_LEN = 512         # frames per clip
MAX_CORPUS = 65536         # clips per corpus
# the fp32 query-vs-frame similarity block of one query chunk stays under this many bytes
_S_BLOCK_BYTES = 256 << 20


class VideoCorpus:
    """A corpus prepared once for ranking: the frames of `embed_video_corpus` L2-normalised into
    split-bf16 halves (the B operand of the similarity GEMM), their inverse norms (to recover the
    raw dot products of the span head) and the frame mask as bytes.

    frame_embeddings: (Nv, L, H) on the GPU; c_attn_masks: (Nv, L)."""

    def __init__(self, frame_embeddings, c_attn_masks):
        if frame_embeddings.dim() != 3 or tuple(c_attn_masks.shape) != frame_embeddings.shape[:2]:
            raise ValueError(f"corpus of shape {tuple(frame_embeddings.shape)} with mask "
                             f"{tuple(c_attn_masks.shape)}: expected (Nv, L, H) and (Nv, L)")
        nv, length, d = frame_embeddings.shape
        if not 1 <= length <= MAX_CLIP_LEN:
            raise ValueError(f"clips of {length} frames: the ranking kernels take 1..{MAX_CLIP_LEN}")
        if not 1 <= nv <= MAX_CORPUS:
            raise ValueError(f"corpus of {nv} clips: the ranking kernels take 1..{MAX_CORPUS}")
        if d % 8:
            raise ValueError(f"hidden size {d} is not a multiple of 8")
        dev = frame_embeddings.device
        frames = frame_embeddings.float().contiguous().view(nv * length, d)
        self.ld = (nv * length + 7) // 8 * 8              # GEMM N (and S row stride): multiple of 8
        self.hi = torch.zeros((self.ld, d), dtype=torch.bfloat16, device=dev)
        self.lo = torch.zeros((self.ld, d), dtype=torch.bfloat16, device=dev)
        self.inv = torch.empty(nv * length, dtype=torch.float32, device=dev)
        ops.l2norm_split(frames, self.hi, self.lo, self.inv)
        self.mask = (c_attn_masks != 0).to(device=dev, dtype=torch.uint8).contiguous()
        self.n_videos, self.length, self.dim, self.device = nv, length, d, dev


def _check_rank_args(corpus, tasks, q2c_alpha, max_video, min_pred_l, max_pred_l, max_before_nms,
                     gt_vidx, kernel_width):
    tasks = tuple(tasks)
    bad = [t for t in tasks if t not in RANK_TASKS]
    if bad or not tasks:
        raise ValueError(f"tasks {tasks}: expected a non-empty subset of {RANK_TASKS}")
    if "VR" in tasks or "VCMR" in tasks:
        if not 1 <= max_video <= min(MAX_SELECT, corpus.n_videos):
            raise ValueError(f"max_video = {max_video}: needs 1 <= max_video <= "
                             f"min({MAX_SELECT}, {corpus.n_videos} clips in the corpus)")
    if "VCMR" in tasks:
        if q2c_alpha is None or q2c_alpha <= 0:
            raise ValueError("VCMR ranks exp(q2c_alpha * score): q2c_alpha must be > 0")
        if max_video * corpus.length * corpus.length >= 1 << 31:
            raise ValueError(f"max_video * L * L = {max_video * corpus.length ** 2} moments per "
                             "query exceeds the kernel's 2^31 limit")
    if "VCMR" in tasks or "SVMR" in tasks:
        if not 1 <= max_before_nms <= MAX_SELECT:
            raise ValueError(f"max_before_nms = {max_before_nms} outside [1, {MAX_SELECT}]")
        if min_pred_l < 0:
            raise ValueError(f"min_pred_l = {min_pred_l} < 0")
        if kernel_width % 2 == 0 or kernel_width > 15:
            raise ValueError(f"span convolution of width {kernel_width}: odd widths <= 15 only")
    if "SVMR" in tasks:
        if gt_vidx is None:
            raise ValueError("SVMR needs gt_vidx, the ground-truth clip of every query")
        if not (torch.is_tensor(gt_vidx) and gt_vidx.is_cuda):     # host values: checked here
            g = np.asarray(gt_vidx.cpu() if torch.is_tensor(gt_vidx) else gt_vidx)
            if g.size and (g.min() < 0 or g.max() >= corpus.n_videos):
                raise ValueError(f"gt_vidx outside [0, {corpus.n_videos})")
    return tasks


@torch.no_grad()
def rank_modularized(corpus, m, p, w_st, w_ed, *, tasks=RANK_TASKS, q2c_alpha=None, max_video=100,
                     min_pred_l=2, max_pred_l=16, max_before_nms=200, gt_vidx=None):
    """Ranking of encoded queries against a `VideoCorpus` (see `rank_queries`).

    m: modularized queries (Nq, H); p = video_query_linear(m) (Nq, H), needed for VCMR / SVMR;
    w_st / w_ed: the span convolution weights. Returns a dict of device tensors:
      "VR":   (scores (Nq, K), clip rows (Nq, K) int32) — exp(q2c_alpha * s) when q2c_alpha is
              given (eval_vcmr.py), s itself otherwise (eval_vr.py);
      "VCMR": (scores (Nq, N), moments (Nq, N, 3) int32 = (clip row, start, end));
      "SVMR": the same on each query's ground-truth clip.
    Moments are ordered by descending score, ties to the lower flat index j*L*L + s*L + e; a query
    with fewer than N band-valid spans is padded with score 0 and moments -1."""
    kw = w_st.numel() if w_st is not None else 1
    tasks = _check_rank_args(corpus, tasks, q2c_alpha, max_video, min_pred_l, max_pred_l,
                             max_before_nms, gt_vidx, kw)
    dev, nv, L, d = corpus.device, corpus.n_videos, corpus.length, corpus.dim
    nq = m.shape[0]
    need_v = "VR" in tasks or "VCMR" in tasks
    need_p = "VCMR" in tasks or "SVMR" in tasks
    if m.shape[1] != d or (need_p and tuple(p.shape) != tuple(m.shape)):
        raise ValueError(f"queries of width {m.shape[1]} against a corpus of width {d}")
    K, N = max_video, max_before_nms
    f32, i32 = torch.float32, torch.int32
    out = {}
    if need_v:
        v_val = torch.empty((nq, K), dtype=f32, device=dev)
        v_idx = torch.empty((nq, K), dtype=i32, device=dev)
        out["VR"] = (v_val, v_idx)
    for t in ("VCMR", "SVMR"):
        if t in tasks:
            out[t] = (torch.empty((nq, N), dtype=f32, device=dev),
                      torch.empty((nq, N, 3), dtype=i32, device=dev))
    if nq == 0:
        return out
    m = m.float().contiguous()
    if need_p:
        p = p.float().contiguous()
        ws = w_st.detach().float().reshape(-1).contiguous()
        we = w_ed.detach().float().reshape(-1).contiguous()
    if "SVMR" in tasks:
        gt = torch.as_tensor(gt_vidx).to(device=dev, dtype=i32, non_blocking=True).reshape(nq)
    # query chunks: [m^ ; p^] rows of one chunk x every corpus frame in fp32 <= _S_BLOCK_BYTES
    rows_per_q = int(need_v) + int(need_p)
    chunk = max(1, min(nq, _S_BLOCK_BYTES // (rows_per_q * corpus.ld * 4)))
    for a in range(0, nq, chunk):
        b = min(nq, a + chunk)
        nc = b - a
        n_rows = rows_per_q * nc
        a_hi = torch.empty((n_rows, d), dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        a_inv = torch.empty(n_rows, dtype=f32, device=dev)
        r_p = nc if need_v else 0                            # first p^ row of the block
        if need_v:
            ops.l2norm_split(m[a:b], a_hi, a_lo, a_inv)
        if need_p:
            ops.l2norm_split(p[a:b], a_hi[r_p:], a_lo[r_p:], a_inv[r_p:])
        s = torch.empty((n_rows, corpus.ld), dtype=f32, device=dev)
        ops.gemm(a_hi, corpus.hi, s, a_lo=a_lo, b_lo=corpus.lo)
        if need_v:
            scores = torch.empty((nc, nv), dtype=f32, device=dev)
            argmax = torch.empty((nc, nv), dtype=i32, device=dev)
            ops.vsm_masked_max(s, corpus.mask, nc, nv, L, scores, argmax)
            ops.rank_topk(scores, nv, K, v_val[a:b], v_idx[a:b],
                          alpha=float(q2c_alpha or 0.0), apply_exp=q2c_alpha is not None)
        if not need_p:
            continue
        q_rows = torch.arange(r_p, r_p + nc, dtype=i32, device=dev)
        pr, pc = [], []
        if "VCMR" in tasks:
            pr.append(q_rows[:, None].expand(nc, K).reshape(-1))
            pc.append(v_idx[a:b].reshape(-1))
        if "SVMR" in tasks:
            pr.append(q_rows)
            pc.append(gt[a:b])
        pair_row, pair_clip = torch.cat(pr), torch.cat(pc)
        st = torch.empty((pair_row.numel(), L), dtype=f32, device=dev)
        ed = torch.empty_like(st)
        ops.vcmr_span_probs(s, pair_row, pair_clip, a_inv, corpus.inv, corpus.mask, ws, we, nv, L,
                            st, ed)
        off = 0
        if "VCMR" in tasks:
            score, mom = out["VCMR"]
            ops.vcmr_moment_topn(st[:nc * K], ed[:nc * K], v_val[a:b], nc, K, L, min_pred_l,
                                 max_pred_l, N, score[a:b], mom[a:b])
            j = mom[a:b, :, 0]
            clip = v_idx[a:b].gather(1, j.clamp(min=0).long())
            mom[a:b, :, 0] = torch.where(j >= 0, clip, j)
            off = nc * K
        if "SVMR" in tasks:
            score, mom = out["SVMR"]
            ops.vcmr_moment_topn(st[off:], ed[off:], None, nc, 1, L, min_pred_l, max_pred_l, N,
                                 score[a:b], mom[a:b])
            j = mom[a:b, :, 0]
            mom[a:b, :, 0] = torch.where(j >= 0, gt[a:b, None].expand_as(j), j)
    return out


@torch.no_grad()
def rank_queries(model, corpus, query_batch, *, tasks=RANK_TASKS, q2c_alpha=None, max_video=100,
                 min_pred_l=2, max_pred_l=16, max_before_nms=200, gt_vidx=None):
    """Ranks one batch of queries against the whole corpus (eval_vcmr.py:232-323 and the SVMR
    block of :326-354; eval_vr.py:223-233), without a host synchronisation.

    query_batch: the reference's eval query batch on the GPU (`query_input_ids`, `query_pos_ids`,
    `query_attn_masks`), with its text plan (plan.attach_plan(..., 'txt') on the host copy) under
    plan.PLAN_KEY; without one the plan is built from the mask, which reads it back to the host.
    The queries are encoded by the model's `encode_txt_inputs(..., attn_layer=q_feat_attn)`.
    tasks: subset of ("VR", "VCMR", "SVMR"). See `rank_modularized` for the outputs.

    Raises ValueError where the reference would fail or the kernels cannot go: max_video > Nv,
    max_video or max_before_nms > 1024, L > 512, SVMR without gt_vidx.

    Deviations from the reference (DESIGN §4 "Retrieval ranking"): ties are ordered
    deterministically (descending score, lower index first) where torch.topk / torch.sort /
    np.argsort leave them unspecified; only band-valid spans are listed (no zero-score filler)."""
    m = model.encode_txt_inputs(query_batch["query_input_ids"], query_batch["query_pos_ids"],
                                query_batch["query_attn_masks"], attn_layer=model.q_feat_attn,
                                plan=query_batch.get(PLAN_KEY))
    tasks = tuple(tasks)
    p = None
    if "VCMR" in tasks or "SVMR" in tasks:
        p = model.video_query_linear(m.to(model.video_query_linear.weight.dtype))
    return rank_modularized(corpus, m, p, model.video_st_predictor.weight,
                            model.video_ed_predictor.weight, tasks=tasks, q2c_alpha=q2c_alpha,
                            max_video=max_video, min_pred_l=min_pred_l, max_pred_l=max_pred_l,
                            max_before_nms=max_before_nms, gt_vidx=gt_vidx)


def _to_host(out):
    """One device->host copy of every result tensor of a batch (bit-cast to int32 and packed)."""
    keys = sorted(out)
    parts, shapes = [], []
    for k in keys:
        for t in out[k]:
            parts.append(t.reshape(-1).view(torch.int32) if t.dtype == torch.float32
                         else t.reshape(-1))
            shapes.append((t.shape, t.dtype))
    flat = torch.cat(parts).cpu()
    res, o = {}, 0
    it = iter(shapes)
    for k in keys:
        vals = []
        for _ in out[k]:
            shape, dtype = next(it)
            n = int(np.prod(shape))
            v = flat[o:o + n]
            o += n
            vals.append((v.view(torch.float32) if dtype == torch.float32 else v).view(shape).numpy())
        res[k] = tuple(vals)
    return res


class _QueryStager:
    """Uploads each host query batch (tensors and text plan) on a side stream through a
    `loader.BatchStager` ring; the current stream waits for the copy before the batch is ranked."""

    def __init__(self, device):
        self._ring = BatchStager(device, depth=2)
        self._cur = torch.cuda.current_stream(device)
        self._slot = None

    def stage(self, host_batch):
        (dev_batch,), ready, self._slot = self._ring.stage(host_batch)
        self._cur.wait_event(ready)
        return dev_batch

    def release(self):
        """After the work that reads the staged batch has been enqueued."""
        self._ring.release(self._slot, self._cur)


def _run_batches(model, corpus, batches, video_ids, rank_kw, want_gt, post=None):
    """Encodes and ranks every query batch; returns (qids, per-batch host results, has_gt).
    `post(out)`, when given, maps each batch's device results to the dict that is copied.
    Data-parallel, the three are gathered from every rank (all_gather_list) and concatenated in
    rank order; has_gt holds when it holds on every rank."""
    local = {vid: i for i, vid in enumerate(video_ids)}
    stager = _QueryStager(corpus.device)
    qids_all, results, has_gt = [], [], want_gt
    was_training = model.training
    model.eval()
    for batch in batches:
        hb = dict(batch)
        qids, vids = hb.pop("qids"), hb.pop("vids")
        targets = hb.pop("targets", None)
        if has_gt and targets is not None and int(targets.min()) < 0:
            has_gt = False                  # eval_vcmr.py:213-216: no GT -> predictions only
        tasks = tuple(t for t in rank_kw["tasks"] if t != "SVMR" or has_gt)
        qb = {k: hb[k] for k in ("query_input_ids", "query_pos_ids", "query_attn_masks")}
        if "SVMR" in tasks:
            qb["gt_vidx"] = torch.tensor([local[v] for v in vids], dtype=torch.int32)
        tb = attach_plan({"input_ids": qb["query_input_ids"], "pos_ids": qb["query_pos_ids"],
                          "attn_masks": qb["query_attn_masks"]}, "txt")
        qb[PLAN_KEY] = tb[PLAN_KEY]             # built on the host: no read-back on the device
        dqb = stager.stage(qb)
        out = rank_queries(model, corpus, dqb, **dict(rank_kw, tasks=tasks),
                           gt_vidx=dqb.get("gt_vidx"))
        stager.release()
        if post is not None:
            out = post(out)
        results.append(_to_host(out) if out else {})
        qids_all.extend(qids)
    if was_training:
        model.train()
    if _data_parallel():        # every rank's queries against the whole corpus, in rank order
        parts = distributed.all_gather_list((qids_all, results, has_gt))
        qids_all = [q for p in parts for q in p[0]]
        results = [r for p in parts for r in p[1]]
        has_gt = all(p[2] for p in parts)
    return qids_all, results, has_gt


def _top_vr(out):
    """`_run_batches`' `post` of the prediction passes: each VR list cut on the device to the
    first 100 clips, the ones the submission lists (eval_vcmr.py:356-360, eval_vr.py:246-249)."""
    if "VR" in out:
        out["VR"] = tuple(t[:, :100] for t in out["VR"])
    return out


def _vcmr_tasks(model, tasks):
    tasks = tuple(t for t in tasks if t in RANK_TASKS)
    if model.lw_neg_ctx == 0 and model.lw_neg_q == 0:          # no q2video scores
        tasks = tuple(t for t in tasks if t == "SVMR")
    if "VR" not in tasks:                                       # VCMR reads the VR selection
        tasks = tuple(t for t in tasks if t != "VCMR")
    return tasks


def full_vcmr_predictions(model, corpus, batches, video_ids, video2idx, *, tasks=RANK_TASKS,
                          q2c_alpha=20.0, max_vcmr_video=100, min_pred_l=2, max_pred_l=16,
                          max_before_nms=200, vfeat_interval=1.5):
    """The ranking half of the reference's full VCMR evaluation (eval_vcmr.py:205-418).

    corpus: a `VideoCorpus` of the frames `embed_video_corpus` returned; batches: the reference's
    full-eval query batches on the HOST (`vcmr_full_eval_collate`: qids, vids, targets and the
    query tensors); video_ids: the clip id of every corpus row; video2idx: the global
    id -> index map. Returns the reference's `eval_res` dict ({"SVMR", "VCMR", "VR"} lists of
    `dict(desc_id, desc, predictions)`, empty ones dropped, plus "video2idx"), which its
    `get_submission_top_n`, NMS and `eval_retrieval` consume unchanged.

    As in the reference, VCMR is produced only together with VR, VR / VCMR only when the model
    has a video-level loss weight, and SVMR only when every batch carries its targets. Flat VCMR
    indices are decoded with the corpus's own L (the reference uses max_clip_len; the two agree
    when the corpus holds a clip of max_clip_len frames); see `rank_queries` for the other stated
    deviations.

    Data-parallel, each rank ranks its own query batches against the whole corpus and every rank
    returns the lists of all ranks' queries, in rank order (eval_vcmr.py:125-134)."""
    tasks = _vcmr_tasks(model, tasks)
    qids, results, has_gt = [], [], False
    if tasks:
        rank_kw = dict(tasks=tasks, q2c_alpha=q2c_alpha, max_video=max_vcmr_video,
                       min_pred_l=min_pred_l, max_pred_l=max_pred_l, max_before_nms=max_before_nms)
        qids, results, has_gt = _run_batches(model, corpus, batches, video_ids, rank_kw,
                                             "SVMR" in tasks, _top_vr)
    return _submission([int(q) for q in qids], results, has_gt, video_ids, video2idx,
                       vfeat_interval, [(t, t) for t in RANK_TASKS])[0]


def full_vr_predictions(model, corpus, batches, video_ids, video2idx, *, max_vr_video=100):
    """The ranking half of the reference's full video-retrieval evaluation (eval_vr.py:198-263):
    the top `max_vr_video` clips of every query by its raw video score, the first 100 of them
    listed as [video_idx, 0, 0, score]. Arguments and result as `full_vcmr_predictions`, also
    when data-parallel: the lists of every rank's queries, in rank order (eval_vr.py:276-293)."""
    rank_kw = dict(tasks=("VR",), q2c_alpha=None, max_video=max_vr_video)
    qids, results, _ = _run_batches(model, corpus, batches, video_ids, rank_kw, False, _top_vr)
    return _submission(qids, results, False, video_ids, video2idx, None, [("VR", "VR")])[0]


# ------------------------------------------------------------------ temporal NMS and TVR metrics
TVR_TASKS = ("VCMR", "SVMR", "VR")          # utils/tvr_standalone_eval.py TASK_TYPES order
RECALL_TOPKS = (1, 5, 10, 100)
MAX_PRED_PER_QUERY = 100
DESC_TYPES = ("v", "t", "vt")


def nms_moments(score, mom, *, nms_thd, n_in, n_out, interval, by_clip):
    """Greedy temporal NMS of ranked moment lists on the device (csrc/nms.cu), with no host
    synchronisation: the post-processing of post_processing_vcmr_nms (by_clip=True: per clip, then
    merged by score) and post_processing_svmr_nms (by_clip=False: one list).

    score (Nq, N) / mom (Nq, N, 3) as `rank_modularized` returns them (clip row, start, end frame;
    descending score; padded with -1). Reads the first n_in entries of each row; spans are in
    seconds of `interval` per frame, as the submission records them. An entry is dropped when its
    IoU with a kept, higher-ranked entry of its group is > nms_thd; at most 100 are kept per group.
    Returns (score (Nq, n_out), mom (Nq, n_out, 3)), padded with 0 / -1."""
    if not 0 <= n_in <= min(MAX_SELECT, score.shape[1]):
        raise ValueError(f"n_in = {n_in} outside [0, min({MAX_SELECT}, {score.shape[1]})]")
    if not 1 <= n_out <= MAX_SELECT:
        raise ValueError(f"n_out = {n_out} outside [1, {MAX_SELECT}]")
    nq, dev = score.shape[0], score.device
    out_s = torch.empty((nq, n_out), dtype=torch.float32, device=dev)
    out_m = torch.empty((nq, n_out, 3), dtype=torch.int32, device=dev)
    ops.temporal_nms(score, mom, n_in, nms_thd, interval, by_clip, n_out, out_s, out_m)
    return out_s, out_m


def _rounded_percentage(x):
    return round(x * 100, 2)                  # get_rounded_percentage


def _pack_lists(lists):
    """Per-query prediction lists -> (vid, st, ed) float32 (n, P) and valid (n, P), the first
    MAX_PRED_PER_QUERY entries of each, as eval_by_task_type reads them."""
    rows = [p[:MAX_PRED_PER_QUERY] for p in lists]
    lens = np.fromiter(map(len, rows), dtype=np.int64, count=len(rows))
    flat = np.array([r[:3] for row in rows for r in row], dtype=np.float32).reshape(-1, 3)
    n, width = len(rows), max(1, int(lens.max(initial=0)))
    valid = np.arange(width)[None, :] < lens[:, None]
    packed = np.zeros((n, width, 3), dtype=np.float32)
    packed[valid] = flat
    return packed[..., 0], packed[..., 1], packed[..., 2], valid


def _pack_ground_truth(items, video2idx, need_ts, use_desc_type):
    """GT dicts -> clip index (n,), spans float32 (n, T, 2) with their mask (n, T), the DiDeMo
    flag (n,) (>= 4 spans: a hit needs 2 overlaps) and the desc type index (n,)."""
    n = len(items)
    gvid = np.array([video2idx[e["vid_name"]] for e in items], dtype=np.int64)
    dtype = np.zeros(n, dtype=np.int64)
    if use_desc_type:
        bad = {e.get("type") for e in items} - set(DESC_TYPES)
        if bad:
            raise ValueError(f"desc types {sorted(map(str, bad))}: expected one of {DESC_TYPES}")
        dtype = np.array([DESC_TYPES.index(e["type"]) for e in items], dtype=np.int64)
    if not need_ts:
        return gvid, None, None, None, dtype
    spans = []
    for e in items:
        if "ts" not in e:
            raise ValueError(f"ground truth of desc_id {e['desc_id']} has no 'ts'")
        ts = np.asarray(e["ts"], dtype=np.float32)
        if ts.shape == (2,):
            ts = ts[None]
        elif not (ts.ndim == 2 and ts.shape[1] == 2 and len(ts) >= 4):
            raise ValueError(f"ground truth 'ts' of desc_id {e['desc_id']} with shape {ts.shape}: "
                             "expected [st, ed] or at least 4 [st, ed] pairs")
        spans.append(ts)
    width = max(len(s) for s in spans) if spans else 1
    gts = np.zeros((n, width, 2), dtype=np.float32)
    on = np.zeros((n, width), dtype=bool)
    for i, s in enumerate(spans):
        gts[i, :len(s)] = s
        on[i, :len(s)] = True
    return gvid, gts, on, on.sum(1) >= 4, dtype


def _task_metrics(task, vid, st, ed, valid, gt, iou_thds, use_desc_type):
    """eval_by_task_type (utils/tvr_standalone_eval.py:86-257) on packed predictions, vectorised
    over queries: float32 predictions and IoU, `>=` each threshold, the same float64 means."""
    gvid, gts, on, didemo, dtype = gt
    matched = valid & (vid == gvid.astype(np.float32)[:, None])       # (n, P)
    metrics, by_type = OrderedDict(), OrderedDict()
    n_type = [np.sum(dtype == t) for t in range(len(DESC_TYPES))]

    def put(key_fmt, hit_of_k, *key_args):
        for k in RECALL_TOPKS:
            metrics[key_fmt.format(*key_args, k)] = _rounded_percentage(np.mean(hit_of_k(k)))
        return hit_of_k

    hits = []                                   # (key prefix, hit_of_k)
    if task == "VR":
        hits.append(("", put("r{}", lambda k: matched[:, :k].any(1))))
    else:
        inter = np.maximum(0, np.minimum(ed[:, :, None], gts[:, None, :, 1])
                           - np.maximum(st[:, :, None], gts[:, None, :, 0]))
        union = np.maximum(ed[:, :, None], gts[:, None, :, 1]) - np.minimum(st[:, :, None],
                                                                            gts[:, None, :, 0])
        iou = np.divide(inter, union, out=np.zeros_like(inter), where=union != 0)
        iou = iou * matched[:, :, None]         # wrong clip: IoU 0
        rank_in_clip = np.cumsum(matched, axis=1)
        for thd in iou_thds:
            ok = (iou >= thd) & on[:, None, :] & valid[:, :, None]             # (n, P, T)
            corr = np.where(didemo[:, None], ok.sum(-1) >= 2, ok[:, :, 0])
            if task == "VCMR":
                fn = (lambda c: lambda k: c[:, :k].any(1))(corr)
            else:                               # SVMR: the first k clip-matched predictions
                fn = (lambda c: lambda k: (c & matched & (rank_in_clip <= k)).any(1))(corr)
            hits.append((f"{thd}-", put("{}-r{}", fn, thd)))
    if use_desc_type:
        with np.errstate(invalid="ignore", divide="ignore"):
            for t, name in enumerate(DESC_TYPES):
                is_t = dtype == t
                for prefix, fn in hits:
                    for k in RECALL_TOPKS:
                        by_type[f"{name}-{prefix}r{k}"] = _rounded_percentage(
                            1.0 * np.sum(np.logical_and(fn(k), is_t)) / n_type[t])
            by_type["desc_type_ratio"] = "v {} t {} vt {}".format(
                *[_rounded_percentage(1.0 * n_type[t] / len(dtype)) for t in range(3)])
    return metrics, by_type


def _metrics(packed_by_task, ground_truth, video2idx, iou_thds, use_desc_type, match_number):
    """eval_retrieval on {task: (desc_ids, vid, st, ed, valid)}."""
    gt_by_id = {e["desc_id"]: e for e in ground_truth}
    out, by_type = OrderedDict(), OrderedDict()
    for task in TVR_TASKS:
        if task not in packed_by_task:
            continue
        desc_ids, vid, st, ed, valid = packed_by_task[task]
        pos = {d: i for i, d in enumerate(desc_ids)}
        if match_number and set(gt_by_id) != set(pos):
            raise ValueError(f"{task}: desc_ids in predictions and ground_truth must match")
        keys = [k for k in gt_by_id if k in pos]
        rows = np.array([pos[k] for k in keys], dtype=np.int64)
        gt = _pack_ground_truth([gt_by_id[k] for k in keys], video2idx, task != "VR",
                                use_desc_type)
        out[task], by_type[task + "_by_type"] = _task_metrics(
            task, vid[rows], st[rows], ed[rows], valid[rows], gt, iou_thds, use_desc_type)
    if use_desc_type:
        out.update(by_type)
    return out


def eval_retrieval(submission, ground_truth, iou_thds=(0.5, 0.7), use_desc_type=True,
                   match_number=True):
    """The reference's `eval_retrieval` (utils/tvr_standalone_eval.py:260-283) for a submission
    ({"VCMR", "SVMR", "VR"} lists of dict(desc_id, predictions) and "video2idx") against
    ground-truth dicts (desc_id, vid_name, ts, type): R@{1,5,10,100} at each IoU threshold over
    the first 100 predictions, equal (not just close) to the reference's OrderedDicts, with
    "<task>_by_type" entries when use_desc_type.

    Precision follows the reference: predictions (clip index included) in float32, IoU in float32
    and 0 for a prediction of the wrong clip, `>=` the threshold; SVMR counts only clip-matched
    predictions; ground truth with at least 4 `ts` pairs (DiDeMo) counts a hit when 2 or more
    overlap. Raises ValueError for `ts` of 2 or 3 pairs, unknown desc types and, under
    match_number, desc_id sets that differ between a task's predictions and the ground truth."""
    packed = {}
    for task in TVR_TASKS:
        if task in submission:
            by_id = {e["desc_id"]: e for e in submission[task]}
            ids = list(by_id)
            packed[task] = (ids, *_pack_lists([by_id[d]["predictions"] for d in ids]))
    return _metrics(packed, ground_truth, submission["video2idx"], iou_thds, use_desc_type,
                    match_number)


def _packed_moments(score, mom, lookup, interval, svmr):
    """Host arrays of one task -> (vid int64, st, ed, score, valid). The list ends at its first
    padded moment (clip row -1). Times in seconds of `interval` per frame: SVMR in float64
    (find_max_triples_from_upper_triangle_product + eval_vcmr.py:346-350), VCMR from float32
    frame indices (eval_vcmr.py:396-400)."""
    valid = mom[..., 0] >= 0
    vid = np.where(valid, lookup[np.maximum(mom[..., 0], 0)], 0)
    if svmr:
        st = mom[..., 1].astype(np.float64) * interval
        ed = (mom[..., 2].astype(np.float64) + 1) * interval
    else:
        st = mom[..., 1].astype(np.float32) * interval
        ed = mom[..., 2].astype(np.float32) * interval + interval
    return vid, st, ed, score, valid


def _records(desc_ids, vid, st, ed, score, valid):
    n = valid.sum(1).tolist()
    vid, st, ed, score = vid.tolist(), st.tolist(), ed.tolist(), score.tolist()
    return [dict(desc_id=d, desc="", predictions=[
        list(r) for r in zip(vid[i][:c], st[i][:c], ed[i][:c], score[i][:c])])
        for i, (d, c) in enumerate(zip(desc_ids, n))]


def _moment_records(score, mom, video_ids, video2idx, interval, svmr):
    """The predictions of one ranked list (score (N,), moments (N, 3)), as `_submission` lists
    them: the same `_packed_moments` / `_records` code on a one-row batch."""
    lookup = np.array([video2idx[v] for v in video_ids], dtype=np.int64)
    packed = _packed_moments(np.asarray(score)[None], np.asarray(mom)[None], lookup, interval, svmr)
    return _records([None], *packed)[0]["predictions"]


def _submission(desc_ids, results, has_gt, video_ids, video2idx, interval, keys):
    """The submission of `_run_batches`' per-batch host results: for each (task, result key) of
    `keys` that has results, the task's list of dict(desc_id, desc, predictions), one per entry of
    `desc_ids`, predictions [video_idx, st, ed, score] ([video_idx, 0, 0, score] for VR); tasks in
    SVMR, VCMR, VR order, empty ones dropped (SVMR also without ground truth), then "video2idx".
    Also returns what `_metrics` scores: {task: (desc_ids, vid, st, ed as float32, valid)}."""
    lookup = np.array([video2idx[v] for v in video_ids], dtype=np.int64)
    sub, packed = {}, {}
    for task, key in keys:
        parts = [r[key] for r in results if key in r]
        if not parts or not desc_ids or (task == "SVMR" and not has_gt):
            continue
        score, mom = (np.concatenate(x) for x in zip(*parts))
        if task == "VR":
            vid = lookup[mom]
            zeros = np.zeros(vid.shape, dtype=np.int64)
            arr = vid, zeros, zeros, score, np.ones(vid.shape, dtype=bool)
        else:
            arr = _packed_moments(score, mom, lookup, interval, task == "SVMR")
        vid, st, ed, score, valid = arr
        sub[task] = _records(desc_ids, *arr)
        packed[task] = (desc_ids, vid.astype(np.float32), np.asarray(st, dtype=np.float32),
                        np.asarray(ed, dtype=np.float32), valid)
    sub = {k: sub[k] for k in ("SVMR", "VCMR", "VR") if k in sub}
    sub["video2idx"] = video2idx
    return sub, packed


def _merge_ground_truth(ground_truth):
    """The ground truth of every rank's queries: each rank's list gathered (all_gather_list) and
    united in rank order, one entry per desc_id (the first seen), so a rank may pass the ground
    truth of its own shard, as the reference's partial_query_data is, or of the whole split. None
    when any rank passes None."""
    parts = distributed.all_gather_list(ground_truth)
    if any(p is None for p in parts):
        return None
    merged = {}
    for part in parts:
        for e in part:
            merged.setdefault(e["desc_id"], e)
    return list(merged.values())


def full_vcmr_eval(model, corpus, batches, video_ids, video2idx, ground_truth, *,
                   tasks=RANK_TASKS, q2c_alpha=20.0, max_vcmr_video=100, min_pred_l=2,
                   max_pred_l=16, max_before_nms=200, max_after_nms=100, nms_thd=0.5,
                   vfeat_interval=1.5, use_desc_type=True):
    """The reference's full VCMR evaluation from ranking to metrics (validate_full_vcmr,
    eval_vcmr.py:205-508): rank every query batch, run NMS on the device, copy both lists to the
    host in the batch's one copy, and score them with `eval_retrieval`'s arithmetic on the packed
    arrays.

    Data-parallel, each rank ranks its own query batches against the whole corpus (see
    `embed_video_corpus` for the sharded corpus pass), the host arrays of all ranks are gathered in
    rank order, and every rank builds the same submissions and computes the metrics once over the
    union. ground_truth is gathered too and united by desc_id: each rank may pass the ground truth
    of its own queries (the reference's partial_query_data) or that of the whole split; if any
    rank passes None there are no metrics. Stated deviation: the reference averages each rank's already rounded percentages
    weighted by its query count (eval_vcmr.py:431-446). The union gives the one-process result
    whatever the number of ranks: the exact recall rounded to 0.01, where the reference's mean of
    rounded values lies within 0.005 points of the same exact recall. (The reference weights the
    "<task>_by_type" entries by the query count too, not by the count of that type.)

    Arguments as `full_vcmr_predictions`, plus ground_truth: the GT dicts of the evaluated queries
    (the reference's partial_query_data), or None. Returns {"submission": the top-max_after_nms
    lists as get_submission_top_n leaves them, "metrics": eval_retrieval of those}; with
    nms_thd != -1 also {"submission_nms": {"video2idx", "SVMR", "VCMR"} after NMS, "metrics_nms"}.
    Metrics are given only when every batch has targets and ground_truth is not None.

    This reproduces what the reference effectively does:
    * get_submission_top_n (eval_vcmr.py:420) truncates the eval_res lists in place, so its NMS
      reads only the first min(max_before_nms, max_after_nms) predictions, not max_before_nms.
    * The same aliasing makes the reference return the post-NMS SVMR / VCMR lists as its
      eval_submission; both are returned here, explicitly.
    * NMS keeps at most 100 moments per clip (the inner default of temporal_non_maximum_suppression)
      whatever max_after_nms is.
    Deviations: those of `full_vcmr_predictions`, and an SVMR query without any band-valid span
    gets an empty list where the reference raises IndexError (tvr_eval_utils.py:231). The
    reference computes the post-NMS lists only when it has ground truth."""
    tasks = _vcmr_tasks(model, tasks)
    if max_after_nms < 1:
        raise ValueError(f"max_after_nms = {max_after_nms} < 1")
    do_nms = nms_thd != -1
    n_top = min(max_before_nms, max_after_nms)
    n_vr = min(100, max_after_nms)

    def post(out):
        res = {}
        if "VR" in out:
            res["VR"] = tuple(t[:, :n_vr] for t in out["VR"])
        for t in ("VCMR", "SVMR"):
            if t in out:
                s, m = out[t]
                res[t] = (s[:, :n_top], m[:, :n_top])
                if do_nms:
                    res[t + "_NMS"] = nms_moments(s, m, nms_thd=nms_thd, n_in=n_top, n_out=n_top,
                                                  interval=vfeat_interval, by_clip=t == "VCMR")
        return res

    qids, results, has_gt = [], [], False
    if tasks:
        rank_kw = dict(tasks=tasks, q2c_alpha=q2c_alpha, max_video=max_vcmr_video,
                       min_pred_l=min_pred_l, max_pred_l=max_pred_l, max_before_nms=max_before_nms)
        qids, results, has_gt = _run_batches(model, corpus, batches, video_ids, rank_kw, True,
                                             post)
    desc_ids = [int(q) for q in qids]

    def build(keys):
        return _submission(desc_ids, results, has_gt, video_ids, video2idx, vfeat_interval, keys)

    if _data_parallel():
        ground_truth = _merge_ground_truth(ground_truth)
    with_metrics = has_gt and ground_truth is not None
    iou_thds = (0.5, 0.7)                      # VCMR_IOU_THDS (utils/const.py)
    out = {}
    out["submission"], packed = build([("SVMR", "SVMR"), ("VCMR", "VCMR"), ("VR", "VR")])
    if with_metrics:
        out["metrics"] = _metrics(packed, ground_truth, video2idx, iou_thds, use_desc_type, True)
    if do_nms:
        out["submission_nms"], packed = build([("SVMR", "SVMR_NMS"), ("VCMR", "VCMR_NMS")])
        if with_metrics:
            out["metrics_nms"] = _metrics(packed, ground_truth, video2idx, iou_thds,
                                          use_desc_type, True)
    return out


def _validate_qa(model, loader, task, save_logits, batch_stats, log_keys):
    """The evaluation loop of validate_videoqa / validate_violin: returns (val_log, results,
    logits). `batch_stats(scores, targets)` gives the batch's device tensors (answers, loss sum,
    correct count, ground-truth flag); they and, with `save_logits`, the scores come back in one
    device->host copy. From the first batch whose flag is negative, only predictions are made,
    and there is no val_log. `log_keys` names its loss, accuracy and rate.

    Data-parallel, one all_gather_list sums the loss, the correct count and the example count over
    ranks, ands the ground-truth flag and unites the results / logits dicts, on every rank. The
    rate is the global count over this rank's wall time."""
    import time
    model.eval()
    val_loss, n_ex, tot_score = 0.0, 0, 0
    results, logits, val_log = {}, {}, {}
    t0 = time.time()
    has_gt = True
    for batch in loader:
        qids = batch.pop("qids")
        targets = batch["targets"]
        scores = model(batch, task, compute_loss=False)
        answers, loss, correct, gt = batch_stats(scores, targets)
        packed = torch.cat([answers.float().reshape(-1), loss.reshape(1).float(),
                            correct.reshape(1).float(), gt.reshape(1).float()] +
                           ([scores.float().reshape(-1)] if save_logits else []))
        host = packed.cpu()
        n = answers.numel()
        b_loss, b_correct, b_gt = (float(x) for x in host[n:n + 3])
        if b_gt < 0:
            has_gt = False
        for qid, answer in zip(qids, host[:n].long().tolist()):
            results[str(qid)] = answer
        if save_logits:
            for qid, row in zip(qids, host[n + 3:].view(n, -1).tolist()):
                logits[str(qid)] = row
        if has_gt:
            val_loss += b_loss
            tot_score += int(b_correct)
            n_ex += len(qids)
    if _data_parallel():
        parts = distributed.all_gather_list((val_loss, tot_score, n_ex, has_gt, results, logits))
        val_loss, tot_score, n_ex = (sum(p[i] for p in parts) for i in range(3))
        has_gt = all(p[3] for p in parts)
        results = {k: v for p in parts for k, v in p[4].items()}
        logits = {k: v for p in parts for k, v in p[5].items()}
    if has_gt:
        tot_time = time.time() - t0
        val_log = {log_keys[0]: val_loss / n_ex, log_keys[1]: tot_score / n_ex,
                   log_keys[2]: n_ex / tot_time}
    model.train()
    return val_log, results, logits


@torch.no_grad()
def validate_videoqa(model, loader, split, task="tvqa", save_logits=False):
    """eval_videoQA.py:120-173 (validate_videoQA): returns (val_log, results, logits) with
    `valid/loss`, `valid/acc`, `valid/ex_per_s`, results[str(qid)] = predicted answer index and,
    with `save_logits`, logits[str(qid)] = the candidate logits. Once a batch carries a negative
    target ("no ground truth") only predictions are made and val_log stays empty, as in the
    reference. Loss sums and correct counts are computed on the device; each batch makes one
    device->host copy (answers, loss sum, correct count, smallest target, logits). `split` names
    the split only.

    Data-parallel, each rank evaluates its own batches; one all_gather_list then sums the loss,
    the correct count and the example count over ranks, and results / logits are the union of
    every rank's dicts (eval_videoQA.py:95-99), on every rank. No ground truth on any rank means no
    val_log on every rank. ex_per_s is the global count over this rank's wall time."""
    def batch_stats(scores, targets):                                    # scores (Nv, Nq)
        tgt = targets.to(scores.device).reshape(-1)
        answers = scores.max(dim=-1)[1]
        loss = torch.nn.functional.cross_entropy(scores, tgt.clamp(min=0), reduction="sum")
        return answers, loss, (answers == tgt).sum(), tgt.min()

    return _validate_qa(model, loader, task, save_logits, batch_stats,
                        ("valid/loss", "valid/acc", "valid/ex_per_s"))


@torch.no_grad()
def validate_violin(model, loader, split, save_logits=False):
    """eval_violin.py:118-164 (validate_violin): returns (val_log, results, logits) with
    `valid/{split}_loss` (summed binary cross entropy of sigmoid(score) over the examples),
    `valid/{split}_acc` and `valid/{split}_ex_per_s`, results[str(qid)] = int(sigmoid(score) > 0.5)
    and, with `save_logits`, logits[str(qid)] = [score]. Predictions, the loss sum and the correct
    count are computed on the device; each batch makes one device->host copy. Unlike the
    reference, a one-row batch works (there `predictions.squeeze().tolist()` is an int and the zip
    over it raises). Data-parallel, the sums and dicts of every rank are merged as in
    `validate_videoqa` (eval_violin.py:94-98)."""
    def batch_stats(scores, targets):                                    # scores (rows, 1)
        tgt = targets.to(scores.device).reshape(scores.shape)
        probs = torch.sigmoid(scores)
        predictions = (probs > 0.5).long()
        loss = torch.nn.functional.binary_cross_entropy(probs, tgt.to(scores.dtype),
                                                        reduction="sum")
        # no "no ground truth" rule in eval_violin.py: a constant flag, not the smallest target
        return predictions, loss, (predictions == tgt).sum(), loss.new_zeros(())

    return _validate_qa(model, loader, "violin", save_logits, batch_stats,
                        tuple(f"valid/{split}_{k}" for k in ("loss", "acc", "ex_per_s")))


# ------------------------------------------------------------------ pretraining validation
# pretrain.py:387-608. Every metric sum stays in a small fp32 device accumulator; each task makes
# ONE device->host copy, after its last batch. Example counts come from host-known shapes.
# Data-parallel, the counts join the sums and the copy reads their sum over ranks (_task_totals).
def _task_totals(acc, counts):
    """The one device->host copy of a validation task: its device sums `acc` and its host
    `counts`, as (list of floats, list of ints). Data-parallel, both go into one fp64 device
    tensor (counts exact up to 2^53) that `distributed.sum_over_ranks` adds up before the copy:
    a rank with no batch still joins, and every division uses the global counts."""
    if not _data_parallel():
        return acc.cpu().tolist(), list(counts)
    dev = acc.device
    both = torch.cat([acc.double()] + [torch.full((1,), float(c), dtype=torch.float64, device=dev)
                                       for c in counts])
    host = distributed.sum_over_ranks(both).cpu().tolist()
    k = acc.numel()
    return host[:k], [int(c) for c in host[k:]]


def attach_mlm_plan(batch):
    """Collate-side hook for MLM batches: plan.attach_plan(batch, "mlm")."""
    return attach_plan(batch, "mlm")


def _f_encoder(model):
    v_enc = model.v_encoder if hasattr(model, "v_encoder") else model
    return v_enc.f_encoder if hasattr(v_enc, "f_encoder") else v_enc


def _device_of(model):
    return next(model.parameters()).device


def _mlm_batch_stats(model, batch, acc):
    """The masked tokens of `batch` through CrossModalTrm.mlm_head_input, then the fused
    vocabulary GEMM with `ops.lm_head_ce_stats`: acc += (sum of the token losses, number of top-1
    hits), and no (n_masked, V) logits tensor."""
    from .params import flat_of
    fe = _f_encoder(model)
    labels = batch["txt_labels"]
    n = int(labels.shape[0])
    if n == 0:
        return 0
    h = fe.mlm_head_input(batch["input_ids"], batch.get("position_ids"), batch.get("v_feat"),
                          batch.get("f_pos_ids"), batch["attn_masks"], batch.get("gather_index"),
                          batch["txt_mask_tgt"], n, batch.get(PLAN_KEY))
    emb = fe.embeddings.word_embeddings.weight
    ops.lm_head_ce_stats(h.to(torch.bfloat16).contiguous(), flat_of(fe, h.device).bf16(emb),
                         fe.lm_head.bias.detach().float().contiguous(),
                         labels.to(device=h.device, dtype=torch.int32), emb.shape[0] - fe.vocab_pad,
                         acc=acc)
    return n


@torch.no_grad()
def validate_mlm(model, val_loader):
    """pretrain.py:436-461: {'loss': summed token cross entropy / n_word, 'acc': top-1 hits /
    n_word, 'tok_per_s'}. Stated deviation: a label tied with another column for the row maximum
    counts as a hit (the reference's torch.max reports one index of the tie)."""
    import time
    t0 = time.time()
    acc = torch.zeros(2, dtype=torch.float32, device=_device_of(model))
    n_word = 0
    for batch in val_loader:
        n_word += _mlm_batch_stats(model, batch, acc)
    (val_loss, n_correct), (n_word,) = _task_totals(acc, [n_word])
    tot_time = time.time() - t0
    return {"loss": val_loss / n_word, "acc": n_correct / n_word, "tok_per_s": n_word / tot_time}


@torch.no_grad()
def validate_mffr(model, val_loader):
    """pretrain.py:464-490: {'loss': sum over masked frames of sqrt(sum (pred - target)^2) /
    n_feat, 'cosine': summed cosine similarity / n_feat, 'feat_per_s'}; both sums come from
    `ops.row_l2_cos`. As in the reference, forward_mfm zeroes the masked frames of the batch's
    c_v_feats in place."""
    import time
    t0 = time.time()
    acc = torch.zeros(2, dtype=torch.float32, device=_device_of(model))
    n_feat = 0
    for batch in val_loader:
        targets = batch["feat_targets"]
        pred = model(batch, task="mffr", compute_loss=False)
        if targets.shape[0]:
            ops.row_l2_cos(pred.float().contiguous(), targets.float().contiguous(), acc=acc)
        n_feat += int(targets.shape[0])
    (val_loss, cosine), (n_feat,) = _task_totals(acc, [n_feat])
    tot_time = time.time() - t0
    return {"loss": val_loss / n_feat, "cosine": cosine / n_feat, "feat_per_s": n_feat / tot_time}


def _nce_batch_stats(pred, pos, neg, acc_ce, acc_l2):
    """MFM-NCE logits pred @ [pos; neg]^T (no temperature, as model.mfm_nce(compute_loss=False))
    through the fused cross-entropy GEMM with labels arange(n): bf16 operands, B zero-padded to a
    multiple of 8 rows that ce_n_valid excludes, no bias. l2 / cosine of pred against pos."""
    n, d = pred.shape
    n_cols = n + neg.shape[0]
    b = torch.zeros(((n_cols + 7) // 8 * 8, d), dtype=torch.bfloat16, device=pred.device)
    b[:n] = pos
    b[n:n_cols] = neg
    labels = torch.arange(n, dtype=torch.int32, device=pred.device)
    ops.lm_head_ce_stats(pred.to(torch.bfloat16).contiguous(), b, None, labels, n_cols, acc=acc_ce)
    ops.row_l2_cos(pred.float().contiguous(), pos.float().contiguous(), acc=acc_l2)


@torch.no_grad()
def validate_mfm_nce(model, val_loader):
    """pretrain.py:493-543: {'loss', 'acc', 'l2', 'cosine', 'feat_per_s'}, every sum divided by
    n_feat. The logits never exist: the fused cross-entropy GEMM keeps online-softmax partials
    and the hit of every row (an exact tie with the label counts as a hit). Its operands are bf16:
    the NCE loss differs from the reference's fp32 logits by the bf16 rounding of pred and of the
    targets (DESIGN §4 "Pretraining validation")."""
    import time
    t0 = time.time()
    dev = _device_of(model)
    acc_ce = torch.zeros(2, dtype=torch.float32, device=dev)
    acc_l2 = torch.zeros(2, dtype=torch.float32, device=dev)
    n_feat = 0
    for batch in val_loader:
        pos = batch["feat_targets"]
        feats, neg_feats = model(batch, task="mfm-nce", compute_loss=False)
        if pos.shape[0]:
            _nce_batch_stats(feats, pos, neg_feats, acc_ce, acc_l2)
        n_feat += int(pos.shape[0])
    (val_loss, n_correct, val_l2, cosine), (n_feat,) = _task_totals(torch.cat([acc_ce, acc_l2]),
                                                                    [n_feat])
    tot_time = time.time() - t0
    return {"loss": val_loss / n_feat, "acc": n_correct / n_feat, "l2": val_l2 / n_feat,
            "cosine": cosine / n_feat, "feat_per_s": n_feat / tot_time}


def _host_mask(plan):
    """The (B, T) clip mask of a ReprPlan, rebuilt on the host from its packed positions."""
    seq = plan.c.seq
    mask = np.zeros((seq.rows, seq.length), dtype=np.int64)
    mask[seq.tok_row, seq.tok_col] = 1
    return torch.from_numpy(mask)


@torch.no_grad()
def validate_fom(model, val_loader):
    """pretrain.py:546-589: {'valid/loss': cross entropy summed over the rows whose target is not
    -1 / their count, 'valid/acc': top-1 hits on those rows / their count, 'valid/ex_per_s'}.
    Unlike the reference (pretrain.py:577-578) the batch is not mutated: `targets` and `vids` are
    left in it. With a plan attached, the temporal pass reads its clip mask from the plan instead
    of the device."""
    import time
    t0 = time.time()
    acc = torch.zeros(3, dtype=torch.float32, device=_device_of(model))
    n_ex = 0
    for batch in val_loader:
        b = {k: v for k, v in batch.items() if k not in ("targets", "vids")}
        if b.get(PLAN_KEY) is not None:
            b["c_attn_masks"] = _host_mask(b[PLAN_KEY])
        scores = model(b, task="fom", compute_loss=False)
        targets = batch["targets"].to(scores.device, non_blocking=True).reshape(scores.shape[0])
        valid = targets != -1
        loss = torch.nn.functional.cross_entropy(scores.float(), targets, ignore_index=-1,
                                                 reduction="sum")
        hits = ((scores.argmax(dim=-1) == targets) & valid).sum()
        acc += torch.stack([loss, hits.float(), valid.sum().float()])
        n_ex += len(batch["vids"])
    (val_loss, tot_score, n_valid_ex), (n_ex,) = _task_totals(acc, [n_ex])
    tot_time = time.time() - t0
    return {"valid/loss": val_loss / n_valid_ex, "valid/acc": tot_score / n_valid_ex,
            "valid/ex_per_s": n_ex / tot_time}


@torch.no_grad()
def validate_vsm(model, val_loader, opts):
    """pretrain.py:409-433: model(batch, 'vsm', compute_loss=True) in eval mode ('sum'
    reductions), the three loss sums accumulated on the device; n_ex = len(q_vidx), the positives
    counted from loss_neg_ctx's shape. Normalised by opts.lw_st_ed / lw_neg_ctx / lw_neg_q as the
    reference does. Data-parallel, the forward takes its in-batch negatives from every rank's
    current batch (val_gather_gpus, as in the reference), so the ranking losses are those of the
    gathered batches and every rank must run the same number of VSM batches: the lengths of loaders
    that have one are compared first, and a difference raises ValueError on every rank (a rank
    that ran out would otherwise leave the others waiting in the gather)."""
    import time
    if _data_parallel():
        lens = distributed.all_gather_list(len(val_loader) if hasattr(val_loader, "__len__")
                                           else None)
        if len(set(lens)) > 1:
            raise ValueError(f"data-parallel VSM validation with {lens} batches on ranks "
                             f"0..{len(lens) - 1}: every rank must run the same number")
    t0 = time.time()
    acc = torch.zeros(3, dtype=torch.float32, device=_device_of(model))
    use_neg = opts.lw_neg_ctx != 0 or opts.lw_neg_q != 0
    n_ex, n_ex_pos = 0, 0
    for batch in val_loader:
        n_ex += len(batch["q_vidx"])
        loss_st_ed, loss_neg_ctx, loss_neg_q = model(batch, "vsm", compute_loss=True)
        parts = [loss_st_ed.sum()]
        if use_neg:
            parts += [loss_neg_ctx.sum(), loss_neg_q.sum()]
            n_ex_pos += loss_neg_ctx.numel()
        acc[:len(parts)] += torch.stack(parts).float()
    (val_loss_st_ed, val_loss_neg_ctx, val_loss_neg_q), (n_ex, n_ex_pos) = _task_totals(
        acc, [n_ex, n_ex_pos])
    tot_time = time.time() - t0
    if opts.lw_st_ed:
        val_loss_st_ed /= n_ex
        val_loss_st_ed /= opts.lw_st_ed
    if n_ex_pos > 0 and opts.lw_neg_q > 0 and opts.lw_neg_ctx > 0:
        val_loss_neg_ctx /= n_ex_pos
        val_loss_neg_q /= n_ex_pos
        val_loss_neg_ctx /= opts.lw_neg_ctx
        val_loss_neg_q /= opts.lw_neg_q
    val_loss = (opts.lw_st_ed * val_loss_st_ed + opts.lw_neg_ctx * val_loss_neg_ctx +
                opts.lw_neg_q * val_loss_neg_q)
    return {"valid/loss_overall": val_loss, "valid/loss_st_ed": val_loss_st_ed,
            "valid/loss_neg_ctx": val_loss_neg_ctx, "valid/loss_neg_q": val_loss_neg_q,
            "valid/ex_per_s": n_ex / tot_time}


def validate_pretrain(model, val_dataloaders, opts):
    """pretrain.py:387-406 (validate): model.eval(), each task's validation chosen by the prefix
    of its name ('mlm', 'mffr', 'mfm-nce', 'fom', 'vsm'), model.train() on exit. Returns the dict
    the reference logs, {f'{task}_{k}': v} over all tasks. `opts` needs lw_st_ed, lw_neg_ctx and
    lw_neg_q. Raises ValueError for an unknown task.

    Data-parallel, each rank validates the batches of its own loaders and every task's sums and
    counts are summed over ranks on the device before the task's one copy, as the reference sums
    them over all_gather_list; every rank returns the same losses and accuracies. The rates
    (tok_per_s, feat_per_s, ex_per_s) are global counts over this rank's wall time."""
    model.eval()
    out = {}
    try:
        for task, loader in val_dataloaders.items():
            if task.startswith("mlm"):
                val_log = validate_mlm(model, loader)
            elif task.startswith("mffr"):
                val_log = validate_mffr(model, loader)
            elif task.startswith("mfm-nce"):
                val_log = validate_mfm_nce(model, loader)
            elif task.startswith("fom"):
                val_log = validate_fom(model, loader)
            elif task.startswith("vsm"):
                val_log = validate_vsm(model, loader, opts)
            else:
                raise ValueError(f"Undefined task {task}")
            out.update({f"{task}_{k}": v for k, v in val_log.items()})
    finally:
        model.train()
    return out


def decode_tvc(model, loader, *, max_step, bos, eos, tokenizer, beam_size=1, length_penalty=0.0,
               min_length=0, no_repeat_ngram_size=0, do_sample=False, temperature=1.0, top_k=0,
               top_p=1.0, seed=0, early_stop=False):
    """inf_tvc.py:83-98 / train_tvc.py:259-283 (decode / validate): greedy captions of every
    segment of every batch (tvc.TvcGenerator, one device->host copy per batch), or with
    `beam_size` > 1 the beam-search captions of TvcGenerator.beam_search (score / len **
    `length_penalty`), or with `do_sample` one sampled caption per segment (TvcGenerator.sample
    with `temperature`, `top_k`, `top_p`), as
    `{'vid_name', 'clip_id', 'ts', 'descs': [{'desc': caption}]}` records, in batch order. The
    tokenizer is any object with `convert_ids_to_tokens` / `convert_tokens_to_string`.
    `min_length` and `no_repeat_ngram_size` apply to every strategy (TvcGenerator), and so does
    `early_stop`: each batch stops decoding once every one of its captions has ended (each rank on
    its own, with no collective inside the loop), with the same captions as without. Batch i of
    rank r samples under tvc.sampling_seed(seed, r, i), so no two batches share their uniforms.
    Data-parallel, every rank returns the records of all ranks, gathered with all_gather_list in
    rank order (train_tvc.py:274). Score them with capeval.TVCEval."""
    from .tvc import TvcGenerator, _check_seed, sampling_seed
    if not float(length_penalty) >= 0.0:
        raise ValueError(f"length_penalty = {length_penalty}: must be >= 0")
    if do_sample and beam_size != 1:
        raise ValueError(f"do_sample with beam_size = {beam_size}: sampling draws one caption per "
                         f"segment and takes beam_size 1")
    _check_seed(seed)
    generator = TvcGenerator(model, max_step, bos, eos, fp16=False, min_length=min_length,
                             no_repeat_ngram_size=no_repeat_ngram_size, early_stop=early_stop)
    model.eval()
    rank = distributed.rank()
    results = []
    for i, batch in enumerate(loader):
        if do_sample:
            outputs = generator.sample(batch, temperature=temperature, top_k=top_k, top_p=top_p,
                                       seed=sampling_seed(seed, rank, i))
        elif beam_size == 1:
            outputs = generator.greedy_decode(batch)
        else:
            outputs = generator.beam_search(batch, beam_size, length_penalty)
        for vid, cid, ts, out_ids in zip(batch["vid_names"], batch["clip_ids"], batch["all_ts"],
                                         outputs):
            output = tokenizer.convert_tokens_to_string(tokenizer.convert_ids_to_tokens(out_ids))
            results.append({"vid_name": vid, "clip_id": cid, "ts": ts,
                            "descs": [{"desc": output}]})
    if _data_parallel():
        results = [r for rs in distributed.all_gather_list(results) for r in rs]
    return results


class ModelSaver(object):
    """utils/save.py:112-130."""

    def __init__(self, output_dir, prefix="model_step", suffix="pt", half=False):
        self.output_dir, self.prefix, self.suffix, self.half = output_dir, prefix, suffix, half

    def save(self, model, step, optimizer=None):
        path = join(self.output_dir, f"{self.prefix}_{step}.{self.suffix}")
        sd = {}
        for k, v in model.state_dict().items():
            v = v.detach().cpu() if isinstance(v, torch.Tensor) else v
            if self.half and isinstance(v, torch.Tensor) and v.dtype == torch.float32:
                v = v.half()          # apex O2 checkpoints of the reference hold fp16 tensors
            sd[k] = v
        sd["vocab_padded"] = any(("word_embeddings.weight" in k or "decoder.weight" in k)
                                 and v.size(0) % 8 == 0 for k, v in sd.items()
                                 if isinstance(v, torch.Tensor))
        torch.save(sd, path)
        if optimizer is not None:
            torch.save({"step": step, "optimizer": _to_cpu(optimizer.state_dict())},
                       f"{self.output_dir}/train_state_{step}.pt")
        return path


def load_checkpoint(model, path_or_state):
    """Loads a reference-style checkpoint (fp16 or fp32 tensors, `vocab_padded` flag) into a
    hero_b200 model that may already have run (the flat bf16 mirror is refreshed)."""
    from .encoder import load_pretrained_weight
    sd = torch.load(path_or_state, map_location="cpu") if isinstance(path_or_state, str) \
        else dict(path_or_state)
    sd.pop("vocab_padded", None)
    sd = {k: (v.float() if isinstance(v, torch.Tensor) and v.dtype == torch.float16 else v)
          for k, v in sd.items()}
    return load_pretrained_weight(model, sd)


def _to_cpu(state):
    if isinstance(state, torch.Tensor):
        return state.detach().cpu()
    if isinstance(state, (list, tuple)):
        return type(state)(_to_cpu(t) for t in state)
    if isinstance(state, dict):
        return {k: _to_cpu(v) for k, v in state.items()}
    return state


class TrainingRestorer(object):
    """utils/save.py:133-181 (two rotating files, resume of model + optimizer + global step)."""

    def __init__(self, output_dir, model, optimizer, save_steps=1000):
        self.save_path = f"{output_dir}/restore.pt"
        self.backup_path = f"{output_dir}/restore_backup.pt"
        self.model, self.optimizer, self.save_steps = model, optimizer, save_steps
        self.global_step = 0
        if exists(self.save_path) or exists(self.backup_path):
            self.restore()

    def step(self):
        self.global_step += 1
        if self.global_step % self.save_steps == 0:
            self.save()

    def save(self):
        ckpt = {"global_step": self.global_step,
                "model_state_dict": _to_cpu(self.model.state_dict()),
                "optim_state_dict": _to_cpu(self.optimizer.state_dict())}
        if exists(self.save_path):
            os.rename(self.save_path, self.backup_path)
        torch.save(ckpt, self.save_path)

    def restore(self):
        try:
            ckpt = torch.load(self.save_path, map_location="cpu")
        except Exception:                                   # noqa: BLE001
            ckpt = torch.load(self.backup_path, map_location="cpu")
        self.global_step = ckpt["global_step"]
        load_checkpoint(self.model, ckpt["model_state_dict"])
        dev = self.optimizer.exp_avg.device
        osd = ckpt["optim_state_dict"]
        osd = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in osd.items()}
        self.optimizer.load_state_dict(osd)
