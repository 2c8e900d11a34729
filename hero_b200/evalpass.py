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
* `validate_videoqa` — eval_videoQA.py:120-173 for one process on HeroForVideoQA.
* `ModelSaver` / `TrainingRestorer` — utils/save.py:112-181 with the same file layout (`vocab_padded`
  flag, `model_step_<n>.pt`, `train_state_<n>.pt`, `restore.pt` + backup), so checkpoints are
  interchangeable with the reference's; optimizer state is FusedAdamW's flat moments.
"""
import os
from collections import OrderedDict
from os.path import exists, join

import numpy as np
import torch

from . import ops
from .loader import BatchStager
from .plan import PLAN_KEY, attach_plan


@torch.no_grad()
def embed_video_corpus(model, batches, n_videos, max_clip_len, device=None, video_indices=None,
                       out_dtype=torch.float32):
    """`batches`: iterable of HOST video batch dicts (reference `video_collate` layout; plans are
    attached here when the collate has not). `video_indices`: per batch the row of each clip in the
    corpus tensors (default: consecutive). Returns (frame_embeddings (n_videos, max_clip_len', H),
    c_attn_masks (n_videos, max_clip_len')) trimmed to the longest clip seen, like the reference."""
    v_enc = model.v_encoder if hasattr(model, "v_encoder") else model
    device = device or next(v_enc.parameters()).device
    was_training = v_enc.training
    v_enc.eval()
    stager = BatchStager(device, depth=3)
    cur = torch.cuda.current_stream(device)
    total, masks, longest, row = None, None, 0, 0
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
        if video_indices is not None:
            idx = torch.as_tensor(video_indices[bi], device=device, dtype=torch.long)
        else:
            idx = torch.arange(row, row + B, device=device)
        total[idx, :T] = emb.to(out_dtype)
        masks[idx, :T] = batch["c_attn_masks"]
        longest = max(longest, T)
        row += B
        bi += 1
    if was_training:
        v_enc.train()
    if total is None:
        return None, None
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
    `post(out)`, when given, maps each batch's device results to the dict that is copied."""
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
    return qids_all, results, has_gt


def _moment_records(score, mom, video_ids, video2idx, interval, svmr):
    recs = []
    keep = mom[:, 0] >= 0                     # padding past the last band-valid span
    score, mom = score[keep], mom[keep]
    if svmr:   # find_max_triples_from_upper_triangle_product + eval_vcmr.py:346-350 (float64)
        st = mom[:, 1].astype(np.float64) * interval
        ed = (mom[:, 2].astype(np.float64) + 1) * interval
    else:      # eval_vcmr.py:396-400 (float32 frame indices)
        st = mom[:, 1].astype(np.float32) * interval
        ed = mom[:, 2].astype(np.float32) * interval + interval
    for i in range(len(score)):
        recs.append([video2idx[video_ids[int(mom[i, 0])]], float(st[i]), float(ed[i]),
                     float(score[i])])
    return recs


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
    deviations."""
    tasks = _vcmr_tasks(model, tasks)
    res = {"SVMR": [], "VCMR": [], "VR": []}
    if tasks:
        rank_kw = dict(tasks=tasks, q2c_alpha=q2c_alpha, max_video=max_vcmr_video,
                       min_pred_l=min_pred_l, max_pred_l=max_pred_l, max_before_nms=max_before_nms)
        qids, results, has_gt = _run_batches(model, corpus, batches, video_ids, rank_kw,
                                             "SVMR" in tasks)
        rows = [(r, i) for r in results for i in range(len(next(iter(r.values()))[0]))]
        assert len(rows) == len(qids)
        for qid, (r, i) in zip(qids, rows):
            if "SVMR" in tasks and has_gt:
                res["SVMR"].append(dict(desc_id=int(qid), desc="", predictions=_moment_records(
                    *(x[i] for x in r["SVMR"]), video_ids, video2idx, vfeat_interval, True)))
            if "VR" in r:
                sc, ix = r["VR"][0][i][:100], r["VR"][1][i][:100]
                res["VR"].append(dict(desc_id=int(qid), desc="", predictions=[
                    [video2idx[video_ids[int(v)]], 0, 0, float(s)] for s, v in zip(sc, ix)]))
            if "VCMR" in r:
                res["VCMR"].append(dict(desc_id=int(qid), desc="", predictions=_moment_records(
                    *(x[i] for x in r["VCMR"]), video_ids, video2idx, vfeat_interval, False)))
    eval_res = {k: v for k, v in res.items() if len(v) != 0}
    eval_res["video2idx"] = video2idx
    return eval_res


def full_vr_predictions(model, corpus, batches, video_ids, video2idx, *, max_vr_video=100):
    """The ranking half of the reference's full video-retrieval evaluation (eval_vr.py:198-263):
    the top `max_vr_video` clips of every query by its raw video score, the first 100 of them
    listed as [video_idx, 0, 0, score]. Arguments and result as `full_vcmr_predictions`."""
    rank_kw = dict(tasks=("VR",), q2c_alpha=None, max_video=max_vr_video)
    qids, results, _ = _run_batches(model, corpus, batches, video_ids, rank_kw, False)
    vr = []
    rows = [(r, i) for r in results for i in range(len(r["VR"][0]))]
    assert len(rows) == len(qids)
    for qid, (r, i) in zip(qids, rows):
        sc, ix = r["VR"][0][i][:100], r["VR"][1][i][:100]
        vr.append(dict(desc_id=qid, desc="", predictions=[
            [video2idx[video_ids[int(v)]], 0, 0, float(s)] for s, v in zip(sc, ix)]))
    eval_res = {k: v for k, v in dict(VR=vr).items() if len(v) != 0}
    eval_res["video2idx"] = video2idx
    return eval_res


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
    """Host arrays of one task -> (vid int64, st, ed, score, valid), times as _moment_records."""
    valid = mom[..., 0] >= 0
    vid = np.where(valid, lookup[np.maximum(mom[..., 0], 0)], 0)
    if svmr:
        st = mom[..., 1].astype(np.float64) * interval
        ed = (mom[..., 2].astype(np.float64) + 1) * interval
    else:
        st = mom[..., 1].astype(np.float32) * interval
        ed = mom[..., 2].astype(np.float32) * interval + interval
    return vid, st, ed, score, valid


def _records(qids, vid, st, ed, score, valid):
    n = valid.sum(1).tolist()
    vid, st, ed, score = vid.tolist(), st.tolist(), ed.tolist(), score.tolist()
    return [dict(desc_id=int(q), desc="", predictions=[
        list(r) for r in zip(vid[i][:c], st[i][:c], ed[i][:c], score[i][:c])])
        for i, (q, c) in enumerate(zip(qids, n))]


def full_vcmr_eval(model, corpus, batches, video_ids, video2idx, ground_truth, *,
                   tasks=RANK_TASKS, q2c_alpha=20.0, max_vcmr_video=100, min_pred_l=2,
                   max_pred_l=16, max_before_nms=200, max_after_nms=100, nms_thd=0.5,
                   vfeat_interval=1.5, use_desc_type=True):
    """The reference's full VCMR evaluation from ranking to metrics (validate_full_vcmr,
    eval_vcmr.py:205-508, one process): rank every query batch, run NMS on the device, copy both
    lists to the host in the batch's one copy, and score them with `eval_retrieval`'s arithmetic
    on the packed arrays.

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
    lookup = np.array([video2idx[v] for v in video_ids], dtype=np.int64)

    def task_arrays(key, svmr):
        parts = [r[key] for r in results if key in r]
        if not parts or (svmr and not has_gt):
            return None
        score, mom = (np.concatenate(x) for x in zip(*parts))
        if key == "VR":
            vid = lookup[mom]
            zeros = np.zeros(vid.shape, dtype=np.int64)
            return vid, zeros, zeros, score, np.ones(vid.shape, dtype=bool)
        return _packed_moments(score, mom, lookup, vfeat_interval, svmr)

    def build(keys):
        sub, packed = {}, {}
        for task, key in keys:
            arr = task_arrays(key, task == "SVMR")
            if arr is None or not qids:
                continue
            vid, st, ed, score, valid = arr
            sub[task] = _records(qids, *arr)
            packed[task] = ([int(q) for q in qids], vid.astype(np.float32),
                            np.asarray(st, dtype=np.float32), np.asarray(ed, dtype=np.float32),
                            valid)
        sub = {k: sub[k] for k in ("SVMR", "VCMR", "VR") if k in sub}
        sub["video2idx"] = video2idx
        return sub, packed

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


@torch.no_grad()
def validate_videoqa(model, loader, split, task="tvqa", save_logits=False):
    """eval_videoQA.py:120-173 (validate_videoQA) for one process: returns (val_log, results,
    logits) with `valid/loss`, `valid/acc`, `valid/ex_per_s`, results[str(qid)] = predicted answer
    index and, with `save_logits`, logits[str(qid)] = the candidate logits. Once a batch carries a
    negative target ("no ground truth") only predictions are made and val_log stays empty, as in
    the reference. Loss sums and correct counts are computed on the device; each batch makes one
    device->host copy (answers, loss sum, correct count, smallest target, logits). Averaging across
    ranks (all_gather_list) is left to the caller. `split` names the split only."""
    import time
    model.eval()
    val_loss, n_ex, tot_score = 0.0, 0, 0
    results, logits, val_log = {}, {}, {}
    t0 = time.time()
    has_gt_target = True
    for batch in loader:
        qids = batch.pop("qids")
        targets = batch["targets"]
        scores = model(batch, task, compute_loss=False)                 # (Nv, Nq)
        tgt = targets.to(scores.device).reshape(-1)
        answers = scores.max(dim=-1)[1]
        loss = torch.nn.functional.cross_entropy(scores, tgt.clamp(min=0), reduction="sum")
        correct = (answers == tgt).sum()
        packed = torch.cat([answers.float(), loss.reshape(1).float(), correct.reshape(1).float(),
                            tgt.min().reshape(1).float()] +
                           ([scores.float().reshape(-1)] if save_logits else []))
        host = packed.cpu()
        n = answers.numel()
        ans = host[:n].long().tolist()
        b_loss, b_correct, b_min = (float(x) for x in host[n:n + 3])
        if has_gt_target and b_min < 0:
            has_gt_target = False
        for qid, answer in zip(qids, ans):
            results[str(qid)] = answer
        if save_logits:
            for qid, row in zip(qids, host[n + 3:].view(n, -1).tolist()):
                logits[str(qid)] = row
        if has_gt_target:
            val_loss += b_loss
            tot_score += int(b_correct)
            n_ex += len(qids)
    if has_gt_target:
        tot_time = time.time() - t0
        val_log = {"valid/loss": val_loss / n_ex, "valid/acc": tot_score / n_ex,
                   "valid/ex_per_s": n_ex / tot_time}
    model.train()
    return val_log, results, logits


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
