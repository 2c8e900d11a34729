"""HeroForViolin (model/violin.py:18-84): VIOLIN video-and-language inference.

Each (video, statement) row of the collate (data/violin.py:63-141) runs the cross-modal
transformer over the video's subtitles with the statement appended, then the temporal transformer
over [frames | statement], then one learned attention pooling of its frame outputs. On this path:

    ReprPlan + QaPlan (host, Nq = 1)  ->  videoqa.encode_query_fused  ->
    qa_pool(w_st=None): softmax over the row's frames + weighted sum  ->  MLPLayer head (torch)

The query-fused pass is video QA's, with the statement rows in place of the question + answer
rows; the pooling is the single-pooling mode of the video QA kernels. The MLPLayer head and the
sigmoid + binary cross entropy stay in torch.
"""
from collections import defaultdict

import torch
from torch import nn
from torch.nn import functional as F

from . import functional as Fn
from .layers import MLPLayer
from .model import HeroModel
from .videoqa import encode_query_fused


class HeroForViolin(HeroModel):
    def __init__(self, config, vfeat_dim, max_frm_seq_len):
        super().__init__(config, vfeat_dim, max_frm_seq_len)
        hsz = config.c_config.hidden_size
        self.violin_pool = nn.Linear(in_features=hsz, out_features=1, bias=False)
        self.violin_pred_head = MLPLayer(hsz, 1)

    def forward(self, batch, task="violin", compute_loss=True):
        """(rows, 1) logits, or with `compute_loss` the mean binary cross entropy of their sigmoid
        against `targets`. Plans attached with plan.attach_plan(kind="violin") are used."""
        batch = defaultdict(lambda: None, batch)
        if task != "violin":
            raise ValueError(f"Unrecognized task: {task}")
        y, qplan, dev = encode_query_fused(self, batch)
        rows, length = qplan.n_videos, qplan.length
        video_masks = batch["c_attn_masks"].float()
        pooled = Fn.qa_pool(y, self.violin_pool.weight, None, dev.frame_map, video_masks, rows, 1,
                            length)
        logits = self.violin_pred_head(pooled.to(self.violin_pred_head.linear_1.weight.dtype))
        if not compute_loss:
            return logits
        # sigmoid then BCE, as the reference: BCE clamps its log at -100, so this differs from
        # binary_cross_entropy_with_logits once the sigmoid saturates
        scores = torch.sigmoid(logits).squeeze(-1)
        targets = batch["targets"].squeeze(-1).to(dtype=scores.dtype)
        return F.binary_cross_entropy(scores, targets, reduction="mean")
