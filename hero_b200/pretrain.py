"""Video-subtitle matching (VSM) / video corpus moment retrieval head on the hero_b200 encoder
(model/pretrain.py:19-413 and model/vcmr.py of the reference; SURVEY.md 8f rank 1).

Same constructor, task names, return values, loss weights and parameter names as the reference
classes, so `train_vcmr.py` / `pretrain.py` and their checkpoints keep working. What differs:

* the video rows and the query rows go through the cross-modal transformer in ONE pass
  (`HierarchicalVlModel.forward_repr_txt`) instead of `v_encoder(batch, 'repr')` followed by
  `v_encoder.f_encoder(query_batch, 'txt')`;
* the cross-rank gather of queries / clips for in-batch negatives uses torch.distributed
  (`distributed.vsm_allgather`, same forward/backward contract as the Horovod-based
  `VsmAllgather`, model/pretrain.py:427-451);
* the head's device work after the query pooling is fused (hero_b200/csrc/vsm.cu): the
  video-level scores are l2norm -> split-bf16 wgmma GEMM -> masked max (3 launches forward, 2
  backward, instead of ~15 + ~25 torch kernels), the span logits one kernel each way; nothing in
  the training-mode forward reads a value back to the host (clips are padded to `max_clip_len`
  for the cross-rank gather instead of exchanging lengths; equal per-rank query / clip counts are
  a stated requirement, `gather_equal_counts`). The ranking losses (two small sorts) stay torch.

Known deviation: hero_b200 returns ZEROS at padded frame positions (packed layout), the reference
returns what its transformer computed there. The width-5 span convolutions reach two frames past
a clip's end, so the start / end logits of the last two valid frames of clips shorter than the
batch maximum differ from the reference's (tests/test_heads_cpu.py pins everything else against
reference outputs, and the span loss on an equal-length batch).
"""
import random
from collections import defaultdict

import torch
from torch import nn
from torch.nn import functional as F

from . import distributed as hdist
from . import functional as Fn
from .encoder import QueryFeatEncoder
from .layers import mask_logits
from .model import HeroModel
from .plan import PLAN_KEY, QUERY_PLAN_KEY


class HeroForPretraining(HeroModel):
    def __init__(self, config, vfeat_dim, max_frm_seq_len, conv_stride=1, conv_kernel_size=5,
                 ranking_loss_type="hinge", margin=0.1, lw_neg_ctx=0, lw_neg_q=0, lw_st_ed=0.01,
                 drop_svmr_prob=0, use_hard_negative=False, hard_pool_size=20,
                 hard_neg_weight=10, use_all_neg=True):
        super().__init__(config, vfeat_dim, max_frm_seq_len)
        self.config = config
        self.lw_st_ed, self.lw_neg_q, self.lw_neg_ctx = lw_st_ed, lw_neg_q, lw_neg_ctx
        self.ranking_loss_type = ranking_loss_type
        self.use_hard_negative = use_hard_negative
        self.hard_pool_size = hard_pool_size
        self.hard_neg_weight = hard_neg_weight
        self.margin = margin
        self.use_all_neg = use_all_neg
        self.drop_svmr_prob = drop_svmr_prob
        self.gather_gpus = True       # in-batch negatives from every rank while training
        # every rank contributes the same number of queries / clips per step (drop_last loaders):
        # the cross-rank gather then needs no count exchange and no host sync. Set False for
        # ragged last batches (falls back to the reference's count exchange, one sync per gather).
        self.gather_equal_counts = True
        self.video_query_linear = nn.Linear(config.q_config.hidden_size,
                                            config.c_config.hidden_size)
        conv = dict(in_channels=1, out_channels=1, kernel_size=conv_kernel_size,
                    stride=conv_stride, padding=conv_kernel_size // 2, bias=False)
        self.video_st_predictor = nn.Conv1d(**conv)
        self.video_ed_predictor = nn.Conv1d(**conv)
        self.qfeat_dim = config.f_config.hidden_size
        self.q_feat_attn = QueryFeatEncoder(config.q_config, self.qfeat_dim)

    # ------------------------------------------------------------------ forward
    def forward(self, batch, task="vsm", compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        if task != "vsm":
            if task.startswith("mlm") or task in ("mffr", "mfm-nce", "fom"):
                return self.v_encoder(batch, task, compute_loss)
            raise ValueError(f"Unrecognized task {task}")
        query_batch = {"input_ids": batch["query_input_ids"], "pos_ids": batch["query_pos_ids"],
                       "attn_masks": batch["query_attn_masks"]}
        if batch[QUERY_PLAN_KEY] is not None:     # collate-side plan (plan.attach_plan(b, 'vsm'))
            query_batch[PLAN_KEY] = batch[QUERY_PLAN_KEY]
        # one cross-modal pass for the clip rows and the query rows
        frame_embeddings, query_tokens = self.v_encoder.forward_repr_txt(batch, query_batch)
        modularized_query = self.q_feat_attn(query_tokens, batch["query_attn_masks"])

        q2video_scores = st_prob = ed_prob = None
        if self.lw_st_ed != 0:
            if random.random() > self.drop_svmr_prob or not self.training:
                st_prob, ed_prob = self.get_pred_from_mod_query(
                    frame_embeddings, batch["c_attn_masks"], modularized_query)
        if self.lw_neg_ctx != 0 or self.lw_neg_q != 0:
            q2video_scores = self.get_video_level_scores(modularized_query, frame_embeddings,
                                                         batch["c_attn_masks"])
        if not compute_loss:
            return q2video_scores, st_prob, ed_prob

        zero = torch.zeros(1, dtype=frame_embeddings.dtype, device=frame_embeddings.device)
        loss_st_ed, loss_neg_ctx, loss_neg_q = zero, zero, zero
        reduction = "mean" if self.training else "sum"
        if st_prob is not None:
            if st_prob.dim() == 3:      # every query against every clip: keep the query's own clip
                rows = torch.arange(len(st_prob), device=st_prob.device)
                st_prob, ed_prob = st_prob[rows, batch["q_vidx"]], ed_prob[rows, batch["q_vidx"]]
            targets = batch["targets"]
            loss_st_ed = (F.cross_entropy(st_prob, targets[:, 0].long(), reduction=reduction,
                                          ignore_index=-1) +
                          F.cross_entropy(ed_prob, targets[:, 1].long(), reduction=reduction,
                                          ignore_index=-1))
        if q2video_scores is not None:
            loss_neg_ctx, loss_neg_q = self.get_video_level_loss(q2video_scores, reduction)
        return (self.lw_st_ed * loss_st_ed, self.lw_neg_ctx * loss_neg_ctx,
                self.lw_neg_q * loss_neg_q)

    # ------------------------------------------------------------------ query side
    def encode_txt_inputs(self, input_ids, pos_ids, attn_masks, attn_layer=None,
                          normalized=False, plan=None):
        """model/pretrain.py:168-186: text-only pass of the cross-modal transformer, optionally
        L2-normalised, optionally pooled by `attn_layer` (the QueryFeatEncoder). `plan`: the
        batch's text plan built on the host (plan.attach_plan(..., 'txt')); without one it is built
        from `attn_masks`, which reads a device mask back to the host."""
        txt = {"input_ids": input_ids, "pos_ids": pos_ids, "attn_masks": attn_masks}
        if plan is not None:
            txt[PLAN_KEY] = plan
        feats = self.v_encoder.f_encoder(txt, "txt")[0]
        if normalized:
            feats = F.normalize(feats, dim=-1, eps=1e-5)
        return feats if attn_layer is None else attn_layer(feats, attn_masks)

    # ------------------------------------------------------------------ span prediction
    def _get_st_ed_prob(self, modularized_query, context_feat2, context_mask, cross=False):
        """Start / end logits per frame: similarity of the projected query to every frame,
        smoothed by a width-5 convolution each (model/pretrain.py:128-166). cross=True scores
        every query against every clip (Nq, Nv, L)."""
        query = self.video_query_linear(modularized_query.to(self.video_query_linear.weight.dtype))
        if not cross:
            # one fused kernel each way: per-frame similarity, both convolutions, mask_logits
            return Fn.vsm_span_logits(query, context_feat2, context_mask,
                                      self.video_st_predictor.weight, self.video_ed_predictor.weight)
        ctx = context_feat2.to(query.dtype)
        sim = torch.einsum("md,nld->mnl", query, ctx)
        n_q, n_c, length = sim.shape
        flat = sim.reshape(n_q * n_c, 1, length)
        st = self.video_st_predictor(flat).view(n_q, n_c, length)
        ed = self.video_ed_predictor(flat).view(n_q, n_c, length)
        mask = context_mask.unsqueeze(0).to(st.dtype)
        return mask_logits(st, mask), mask_logits(ed, mask)

    def get_pred_from_mod_query(self, frame_embeddings, c_attn_masks, modularized_query,
                                cross=False):
        cross = cross or frame_embeddings.shape[0] != modularized_query.shape[0]
        return self._get_st_ed_prob(modularized_query, frame_embeddings, c_attn_masks, cross=cross)

    # ------------------------------------------------------------------ video-level ranking
    def get_video_level_scores(self, modularized_query, context_feat1, context_mask,
                               val_gather_gpus=True):
        """(Nq, Nv) cosine score of every query against every clip = max over the clip's valid
        frames (model/pretrain.py:364-413). Queries / clips of all ranks are gathered first
        (clips padded to the longest) so every rank sees the same in-batch negatives."""
        q, ctx = modularized_query.float(), context_feat1.float()
        gather = (self.training and self.gather_gpus) or (not self.training and val_gather_gpus)
        if gather and hdist.size() > 1:
            # every rank pads its clips to the model's max_clip_len: the gathered block has a
            # known shape and no length exchange (and no device->host read) is needed
            cap = getattr(self.v_encoder, "max_clip_len", ctx.shape[1])
            equal = self.gather_equal_counts and ctx.shape[1] <= cap
            if equal:
                pad = cap - ctx.shape[1]
            else:
                lens = torch.tensor([ctx.shape[1]], device=ctx.device)
                all_lens = [torch.zeros_like(lens) for _ in range(hdist.size())]
                torch.distributed.all_gather(all_lens, lens)
                pad = int(max(int(x) for x in all_lens)) - ctx.shape[1]
            if pad:
                ctx = F.pad(ctx, (0, 0, 0, pad))
                context_mask = F.pad(context_mask, (0, pad))
            q = hdist.vsm_allgather(q, None, equal).contiguous()
            ctx = hdist.vsm_allgather(ctx, None, equal).contiguous()
            context_mask = hdist.vsm_allgather(context_mask, None, equal).contiguous()
        # normalise (F.normalize, eps 1e-5) + einsum("md,nld->mln") + mask_logits + max over frames
        return Fn.vsm_video_scores(q, ctx, context_mask)

    def get_video_level_loss(self, query_context_scores, reduction="mean"):
        """Ranking losses of the positive (query, clip) pairs against negative clips and negative
        queries (model/pretrain.py:203-292). Queries are grouped by clip: rows
        [i * k, (i + 1) * k) belong to clip i, k = Nq / Nv."""
        n_q, n_v = query_context_scores.shape
        k = n_q // n_v
        zero = query_context_scores.new_zeros(())          # (no host->device copy: sync-free)
        if n_v == 1:
            return zero, zero
        rows = torch.arange(n_q, device=query_context_scores.device)
        own = rows // k                                        # the clip of every query
        pos = query_context_scores[rows, own]                  # (Nq,)
        own_mask = own[:, None] == torch.arange(n_v, device=own.device)[None, :]
        masked = query_context_scores.masked_fill(own_mask, 999.0)   # sorts first, then skipped
        pos_by_video = pos.view(n_v, k)                        # (Nv, k)
        video_major = masked.transpose(0, 1)                   # (Nv, Nq)
        if self.use_all_neg:
            neg_ctx = self.get_all_neg_scores(masked, sample_min_idx=1)            # (Nq, Nv-1)
            loss_ctx = self._weight_hard(self.get_ranking_loss(pos.view(n_q, 1), neg_ctx))
            neg_q = self.get_all_neg_scores(video_major, sample_min_idx=k)         # (Nv, Nq-k)
            loss_q = self.get_ranking_loss(pos_by_video.unsqueeze(-1), neg_q.unsqueeze(1))
            loss_q = self._weight_hard(loss_q.view(-1, loss_q.size(2)))            # (Nq, Nq-k)
        else:
            neg_ctx = self.get_sampled_neg_scores(masked, sample_min_idx=1).unsqueeze(-1)
            loss_ctx = self.get_ranking_loss(pos.view(n_q, 1), neg_ctx)
            neg_q = self.get_sampled_neg_scores(video_major, sample_min_idx=k).unsqueeze(-1)
            loss_q = self.get_ranking_loss(pos_by_video, neg_q)
        if reduction == "sum":
            return loss_ctx.mean(1), loss_q.mean(1)
        if reduction == "mean":
            return loss_ctx.mean(1).mean(0), loss_q.mean(1).mean(0)
        if reduction is None:
            return loss_ctx, loss_q
        raise NotImplementedError(f"reduction {reduction} not supported")

    def _weight_hard(self, loss):
        """Hard-negative re-weighting of sorted negatives (the first `hard_pool_size` columns are
        the hardest): x hard_neg_weight for those, x 0.1 for the rest."""
        if not self.use_hard_negative:
            return loss
        w = torch.full_like(loss, 0.1)
        w[:, :self.hard_pool_size] = self.hard_neg_weight
        return w * loss

    def get_sampled_neg_scores(self, scores_masked, sample_min_idx=1):
        """One random negative per row, drawn from the sorted scores after the masked positives
        (from the `hard_pool_size` hardest when hard negatives are on)."""
        n, width = scores_masked.shape
        assert width > sample_min_idx, "Unable to sample negative when bsz==sample_min_idx"
        order = torch.sort(scores_masked, descending=True, dim=1).indices
        hi = min(sample_min_idx + self.hard_pool_size, width) if self.use_hard_negative else width
        pick = torch.randint(sample_min_idx, hi, size=(n,), device=scores_masked.device)
        rows = torch.arange(n, device=scores_masked.device)
        return scores_masked[rows, order[rows, pick]]

    def get_all_neg_scores(self, scores_masked, pos_indices=None, sample_min_idx=1):
        """Every negative per row, hardest first: sorted scores minus the `sample_min_idx` masked
        positives at the front."""
        assert scores_masked.shape[1] > sample_min_idx, (
            "Unable to sample negative when bsz==sample_min_idx")
        return torch.sort(scores_masked, descending=True, dim=1).values[:, sample_min_idx:]

    def get_ranking_loss(self, pos_score, neg_score):
        if self.ranking_loss_type == "hinge":
            return torch.clamp(self.margin + neg_score - pos_score, min=0)
        if self.ranking_loss_type == "lse":
            return torch.log1p(torch.exp(neg_score - pos_score))
        raise NotImplementedError("Only support 'hinge' and 'lse'")

    def set_hard_negative(self, use_hard_negative, hard_pool_size, hard_neg_weight):
        self.use_hard_negative = use_hard_negative
        self.hard_pool_size = hard_pool_size
        self.hard_neg_weight = hard_neg_weight

    def set_train_st_ed(self, lw_st_ed):
        self.lw_st_ed = lw_st_ed


class HeroForVcmr(HeroForPretraining):
    """model/vcmr.py: TVR / How2R / DiDeMo moment retrieval = the VSM head under task names."""

    def forward(self, batch, task="tvr", compute_loss=True):
        if task in ("tvr", "how2r", "didemo_video_sub", "didemo_video_only"):
            return super().forward(batch, task="vsm", compute_loss=compute_loss)
        raise ValueError(f"Unrecognized task {task}")

    def get_pred_from_raw_query(self, frame_embeddings, c_attn_masks, query_input_ids,
                                query_pos_ids, query_attn_masks, cross=False,
                                val_gather_gpus=False):
        modularized_query = self.encode_txt_inputs(query_input_ids, query_pos_ids,
                                                   query_attn_masks, attn_layer=self.q_feat_attn)
        st_prob, ed_prob = self.get_pred_from_mod_query(frame_embeddings, c_attn_masks,
                                                        modularized_query, cross=cross)
        q2video_scores = None
        if self.lw_neg_ctx != 0 or self.lw_neg_q != 0:
            q2video_scores = self.get_video_level_scores(modularized_query, frame_embeddings,
                                                         c_attn_masks, val_gather_gpus)
        return q2video_scores, st_prob, ed_prob


class HeroForVr(HeroForVcmr):
    """model/vr.py: MSR-VTT video retrieval (with or without subtitles) = the VCMR head with the
    span loss off; trains on the video-level ranking losses only. Full-corpus ranking for its
    evaluation is `evalpass.full_vr_predictions`."""

    def __init__(self, config, vfeat_dim, max_frm_seq_len, ranking_loss_type="hinge", margin=0.1,
                 lw_neg_ctx=1, lw_neg_q=1, use_hard_negative=False, hard_pool_size=20,
                 hard_neg_weight=10, use_all_neg=True):
        assert lw_neg_ctx != 0 or lw_neg_q != 0, \
            "Need to set lw_neg_ctx or lw_neg_q for VR training"
        super().__init__(config, vfeat_dim, max_frm_seq_len, ranking_loss_type=ranking_loss_type,
                         margin=margin, lw_neg_ctx=lw_neg_ctx, lw_neg_q=lw_neg_q, lw_st_ed=0,
                         drop_svmr_prob=1.0, use_hard_negative=use_hard_negative,
                         hard_pool_size=hard_pool_size, hard_neg_weight=hard_neg_weight,
                         use_all_neg=use_all_neg)
        assert self.lw_st_ed == 0, "For VR, lw_st_ed should be 0"

    def forward(self, batch, task="msrvtt_video_sub", compute_loss=True):
        if task not in ("msrvtt_video_sub", "msrvtt_video_only"):
            raise ValueError(f"Unrecognized task {task}")
        if compute_loss:
            _, loss_neg_ctx, loss_neg_q = super().forward(batch, task="tvr", compute_loss=True)
            return loss_neg_ctx, loss_neg_q
        q2video_scores, _, _ = super().forward(batch, task="tvr", compute_loss=False)
        return q2video_scores

    def get_pred_from_raw_query(self, frame_embeddings, c_attn_masks, query_input_ids,
                                query_pos_ids, query_attn_masks, cross=False,
                                val_gather_gpus=False):
        """Video scores only (Nq, Nv), from unnormalised query features (model/vr.py:44-56)."""
        modularized_query = self.encode_txt_inputs(query_input_ids, query_pos_ids,
                                                   query_attn_masks, attn_layer=self.q_feat_attn,
                                                   normalized=False)
        return self.get_video_level_scores(modularized_query, frame_embeddings, c_attn_masks,
                                           val_gather_gpus)
