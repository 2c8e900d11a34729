"""HeroForVideoQA (model/videoQA.py:21-112): TVQA / How2QA multiple-choice video QA.

Each (video, candidate answer) row of the collate (data/videoQA.py:62-182) runs the cross-modal
transformer over the video's subtitles with the question and answer appended, then a temporal
transformer over [frames | question + answer], then two learned attention poolings of its frame
outputs. On this path:

    ReprPlan + QaPlan (host)  ->  repr_packed(encode_clip=False) -> qa_fused_embed ->
    c_encoder layers over the query-fused rows -> qa_pool  ->  MLPLayer heads (torch)

Nothing is padded and nothing is concatenated: the frame and question / answer embeddings are
written straight into one packed buffer, and the pooling kernels read the frame rows through the
plan's (video, candidate, frame) -> packed-row map. The two MLPLayer heads, mask_logits on the
start / end logits and the three cross entropies stay in torch, like the MFM / FOM heads.
"""
import copy
from collections import defaultdict

from torch import nn
from torch.nn import functional as F

from . import functional as Fn
from .layers import MLPLayer, mask_logits
from .model import HeroModel
from .plan import PLAN_KEY, QA_PLAN_KEY, ReprPlan, qa_plan

TASKS = ("tvqa", "how2qa")


class HeroForVideoQA(HeroModel):
    def __init__(self, config, vfeat_dim, max_frm_seq_len):
        super().__init__(config, vfeat_dim, max_frm_seq_len)
        hsz = config.c_config.hidden_size
        self.qa_pool = nn.Linear(in_features=hsz, out_features=1, bias=False)
        self.qa_pred_head = MLPLayer(hsz, 1)
        self.st_ed_pool = copy.deepcopy(self.qa_pool)
        self.st_ed_pred_head = MLPLayer(hsz, 2)

    def plans(self, batch):
        """(ReprPlan, QaPlan) of the batch: the attached ones (plan.attach_plan(kind="videoqa")),
        else built here from the masks and question / answer ids (one host read)."""
        rplan, qplan = batch[PLAN_KEY], batch[QA_PLAN_KEY]
        if rplan is None:
            rplan = ReprPlan(batch)
        if qplan is None:
            qplan = qa_plan(batch)
        return rplan, qplan

    def encode_query_fused(self, batch, rplan, qplan):
        """Packed fp32 temporal-transformer outputs of every query-fused row (model/videoQA.py:
        64-82) and the QaPlan's device index."""
        ve = self.v_encoder
        g, _ = ve.repr_packed(batch, rplan, encode_clip=False)
        dev = qplan.to(g.device)
        ce, fe = ve.c_encoder, ve.f_encoder
        # its own dropout stream: a fresh base key, drawn apart from the cross-modal pass's
        drop = ce.encoder.dropout_state()
        ee, te = ce.embeddings, fe.embeddings
        # dropout after each LayerNorm at its own module's rate (FrameEmbeddings of c_config,
        # SubEmbeddings of f_config: model/videoQA.py:70-74)
        cfg = {"drop": drop, "frm_p": ee.dropout.p if self.training else 0.0,
               "qa_p": te.dropout.p if self.training else 0.0,
               "n_tok": qplan.seq.n_tok, "n_frm": qplan.n_frm, "n_qa": qplan.n_qa,
               "frm_tok": dev.frm_tok, "frm_t": dev.frm_t, "qa_tok": dev.qa_tok,
               "qa_ids": dev.qa_ids, "qa_pos": dev.qa_pos, "cpos_off": dev.cpos_off,
               "cpos_idx": dev.cpos_idx, "qpos_off": dev.qpos_off, "qpos_idx": dev.qpos_idx,
               "pad_idx": te.padding_idx}
        emb, emb32 = Fn.qa_fused_embed(g, cfg, [
            ee.position_embeddings.weight, ee.LayerNorm.weight, ee.LayerNorm.bias,
            te.word_embeddings.weight, te.position_embeddings.weight,
            te.token_type_embeddings.weight, te.LayerNorm.weight, te.LayerNorm.bias])
        y = ce.encoder.forward_packed(emb, qplan.attn(dev), drop, x_f32=emb32, out_f32=True)
        return y, dev

    def forward(self, batch, task="tvqa", compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        if task not in TASKS:
            raise ValueError(f"Unrecognized task: {task}")
        targets = batch["targets"].squeeze(-1)
        c_attn_masks = batch["c_attn_masks"]
        rplan, qplan = self.plans(batch)
        y, dev = self.encode_query_fused(batch, rplan, qplan)
        nv, nq, length = qplan.n_videos, qplan.n_cand, qplan.length
        video_masks = c_attn_masks.view(nv, nq, length).float()
        qa_pooled, st_ed_pooled = Fn.qa_pool(y, self.qa_pool.weight, self.st_ed_pool.weight,
                                             dev.frame_map, video_masks, nv, nq, length)
        wdt = self.qa_pred_head.linear_1.weight.dtype
        pred_st_ed = self.st_ed_pred_head(st_ed_pooled.view(nv, length, -1).to(wdt))
        st_prob = mask_logits(pred_st_ed[:, :, 0], video_masks[:, 0])
        ed_prob = mask_logits(pred_st_ed[:, :, 1], video_masks[:, 0])
        logits = self.qa_pred_head(qa_pooled.view(nv, nq, -1).to(wdt)).squeeze(-1)
        if not compute_loss:
            return logits
        ts_targets = batch["ts_targets"]
        st_loss = F.cross_entropy(st_prob, ts_targets[:, 0], reduction="mean", ignore_index=-1)
        ed_loss = F.cross_entropy(ed_prob, ts_targets[:, 1], reduction="mean", ignore_index=-1)
        temporal_loss = (st_loss + ed_loss) / 2.
        qa_loss = F.cross_entropy(logits, targets, reduction="mean", ignore_index=-1)
        return qa_loss, temporal_loss
