"""HierarchicalVlModel / HeroModel with the reference's API (model/model.py:117-364).

`forward_repr` is the hot path of BASELINE.json: cross-modal transformer over per-subtitle
{frames, tokens}, frame outputs merged back onto the clip timeline, residual with the projected
raw frame features, temporal transformer. It runs packed end to end:

    plan (host, numpy)  ->  cross_modal_embed -> 6 x layer -> frame_merge -> frame_embed ->
    3 x layer -> unpack to (B, T, H)

The python double loop of collect_frame_outputs (640 iterations with an H2D copy each on the
canonical batch, model/model.py:171-186) is one CSR gather-sum kernel.
"""
import json
from collections import defaultdict

import torch
from torch import nn
from torch.nn import functional as F

from . import functional as Fn
from .encoder import (CrossModalTrm, RobertaModelConfig, RobertaPreTrainedModel, TemporalTrm,
                      load_pretrained_weight)
from .layers import GELU, BertLayerNorm, LinearLayer, MLPLayer
from .params import flat_of
from .plan import PLAN_KEY, JointPlan, ReprPlan, TxtPlan, plan_inputs

BF16 = torch.bfloat16


class VideoModelConfig(object):
    """model/model.py:31-61."""

    def __init__(self, config_json_file):
        assert isinstance(config_json_file, str)
        with open(config_json_file, "r", encoding="utf-8") as reader:
            config = json.loads(reader.read())
        self.f_config = RobertaModelConfig.from_dict(config["f_config"])
        self.c_config = RobertaModelConfig.from_dict(config["c_config"])
        self.q_config = (RobertaModelConfig.from_dict(config["q_config"])
                         if "q_config" in config else None)
        self.d_config = (RobertaModelConfig.from_dict(config["d_config"])
                         if "d_config" in config else None)
        self.initializer_range = self.f_config.initializer_range

    @classmethod
    def from_json_file(cls, json_file):
        return VideoModelConfig(json_file)


class VideoPreTrainedModel(RobertaPreTrainedModel):
    """model/model.py:64-101."""

    def __init__(self, config, *inputs, **kwargs):
        if not isinstance(config, VideoModelConfig):
            raise ValueError(
                "Parameter config in `{}(config)` should be an instance of class "
                "`VideoModelConfig`.".format(self.__class__.__name__))
        super().__init__(config.f_config)
        self.config = config

    @classmethod
    def load_config(cls, config_file):
        return VideoModelConfig.from_json_file(config_file)

    @classmethod
    def from_pretrained(cls, config_file, state_dict, *inputs, **kwargs):
        config = cls.load_config(config_file)
        model = cls(config, *inputs, **kwargs)
        if state_dict == {}:
            return model
        return load_pretrained_weight(model, state_dict)


class FrameFeatureRegression(nn.Module):
    """model/model.py:104-114 (MFM head, 'next' row): torch ops on the few masked frames."""

    def __init__(self, hidden_size, feat_dim):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(hidden_size, hidden_size), GELU(),
                                 BertLayerNorm(hidden_size, eps=1e-5),
                                 nn.Linear(hidden_size, feat_dim))

    def forward(self, input_):
        return self.net(input_)


class HierarchicalVlModel(VideoPreTrainedModel):
    def __init__(self, config, vfeat_dim, max_frm_seq_len, max_clip_len=100, nce_temp=1.0):
        super().__init__(config)
        self.f_encoder = CrossModalTrm(config.f_config, vfeat_dim, max_frm_seq_len)
        self.frame_transform = LinearLayer(vfeat_dim, config.f_config.hidden_size, layer_norm=True,
                                           dropout=config.f_config.hidden_dropout_prob, relu=True)
        self.c_encoder = TemporalTrm(config.c_config)
        self.feat_regress = FrameFeatureRegression(config.f_config.hidden_size, vfeat_dim)
        self.nce_temp = nce_temp
        self.max_clip_len = max_clip_len
        self.mask_embedding = nn.Embedding(2, vfeat_dim, padding_idx=0)
        self.fom_output = MLPLayer(config.c_config.hidden_size, max_clip_len)
        self.register_buffer("pad", torch.zeros(8, config.c_config.hidden_size))
        self.output_dtype = torch.float32

    def forward(self, batch, task="repr", compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        if task == "repr":
            return self.forward_repr(batch)
        elif task.startswith("mlm"):
            return self.f_encoder(batch, task, compute_loss)
        elif task == "mffr":
            return self.forward_mfm(batch, compute_loss, loss="regression")
        elif task == "mfm-nce":
            return self.forward_mfm(batch, compute_loss, loss="nce")
        elif task == "fom":
            return self.forward_fom(batch, compute_loss)
        else:
            raise ValueError(f"Unrecognized task {task}")

    # ------------------------------------------------------------------ packed hot path
    def _plan(self, batch):
        plan = batch[PLAN_KEY]
        if plan is None:
            plan = ReprPlan(plan_inputs(batch))   # reads masks and ids back in one copy
        return plan

    def repr_packed(self, batch, plan, encode_clip=True, txt_batch=None, txt_plan=None):
        """Returns (packed clip-level tensor bf16 [n_c_tokens, H], dev[, packed query rows]).
        With `txt_batch` the text-only query rows ride through the cross-modal transformer in the
        same pass as the video rows (plan.JointPlan)."""
        device = batch["c_v_feats"].device
        dev = plan.to(device)
        flat = flat_of(self, device)
        fe, ce = self.f_encoder, self.c_encoder
        drop = fe.encoder.dropout_state()
        yq = None
        shared = batch["c_v_feats"] if batch["f_v_feats"] is None else None
        if txt_batch is None:
            # cross-modal transformer on packed [frames, text] rows
            hf = fe.encode_packed(plan.f, dev, plan.f.seq.attn(dev, "f_"), batch["f_v_feats"],
                                  batch["f_v_masks"], drop, shared_feats=shared)
        else:
            jplan = plan.__dict__.get("_joint")
            if jplan is None or jplan.t is not txt_plan:
                jplan = JointPlan(plan, txt_plan)
                plan.__dict__["_joint"] = jplan
            jdev = jplan.to(device)
            y = fe.encode_packed(jplan, jdev, jplan.attn(jdev), batch["f_v_feats"],
                                 batch["f_v_masks"], drop, shared_feats=shared)
            hf, yq = y[:jplan.n_video_tok], y[jplan.n_video_tok:]
        # frame outputs back onto the clip timeline + projected raw features (residual)
        c_v = batch["c_v_feats"]
        D = c_v.shape[-1]
        feats = c_v.reshape(-1, D)
        if feats.dtype != torch.float32:
            feats = feats.float()
        ft = self.frame_transform
        drop_ft = Fn.DropoutState(ft.net[0].p, 0.0, self.training, drop.base + 7919)
        cfg = {"drop": drop_ft, "n_tok": plan.c.seq.n_tok, "n_f_tok": plan.f.seq.n_tok,
               "fwd_off": dev.c_fwd_off, "fwd_idx": dev.c_fwd_idx, "bwd_off": dev.c_bwd_off,
               "bwd_idx": dev.c_bwd_idx, "feats": feats.contiguous(), "src": dev.c_src,
               "lin_w_bf16": flat.bf16(ft.net[1].weight)}
        g = Fn.frame_merge(hf, cfg, [ft.LayerNorm.weight, ft.LayerNorm.bias, ft.net[1].weight,
                                     ft.net[1].bias])
        if not encode_clip:
            return (g, dev) if txt_batch is None else (g, dev, yq)
        dropc = ce.encoder.dropout_state(drop.base + 104729)
        y = ce.embed_encode_packed(g, dev.c_t, plan.c.seq.attn(dev, "c_"), dev.c_pos_off,
                                   dev.c_pos_idx, dropc)
        return (y, dev) if txt_batch is None else (y, dev, yq)

    def _unpack_c(self, y, dev, shape):
        out = Fn.gather_rows(y, dev.c_pad_to_tok, dev.c_tok_flat)
        out = out.view(shape[0], shape[1], y.shape[1])
        return out if out.dtype == self.output_dtype else out.to(self.output_dtype)

    def forward_repr(self, batch, encode_clip=True):
        """model/model.py:195-224 -> (B, T, H); padded frames hold zeros."""
        if not isinstance(batch, defaultdict):
            batch = defaultdict(lambda: None, batch)
        plan = self._plan(batch)
        y, dev = self.repr_packed(batch, plan, encode_clip)
        return self._unpack_c(y, dev, plan.shape_c)

    def forward_repr_txt(self, batch, txt_batch, encode_clip=True):
        """Fused equivalent of
            clip = self.forward_repr(batch);  q = self.f_encoder(txt_batch, 'txt')[0]
        (model/pretrain.py:65-70, model/model.py:226-237): the query rows share the cross-modal
        transformer pass of the video rows. Returns (clip_outputs (B,T,H), query seq (Nq,Lq,H))."""
        if not isinstance(batch, defaultdict):
            batch = defaultdict(lambda: None, batch)
        plan = self._plan(batch)
        tplan = txt_batch.get(PLAN_KEY) if hasattr(txt_batch, "get") else None
        if tplan is None:
            tplan = TxtPlan(**plan_inputs(txt_batch, "txt"))
        y, dev, yq = self.repr_packed(batch, plan, encode_clip, txt_batch, tplan)
        clip = self._unpack_c(y, dev, plan.shape_c)
        tdev = tplan.to(y.device)
        q = Fn.gather_rows(yq.contiguous(), tdev.f_pad_to_tok, tdev.f_tok_flat)
        q = q.view(tplan.shape[0], tplan.shape[1], y.shape[1]).to(self.output_dtype)
        return clip, q

    def collect_frame_outputs(self, out_shape, frame_sequence_output, num_subs,
                              sub_idx2frame_idx):
        """API-compatible restatement of model/model.py:156-187 as ONE index_add (no python
        loop over subtitles); the packed path never calls it."""
        B, T, H = out_shape
        rows, ks, dst = [], [], []
        start = 0
        for vid, n_sub in enumerate(num_subs):
            for sid, frames in sub_idx2frame_idx[vid]:
                rows.extend([start + sid] * len(frames))
                ks.extend(range(len(frames)))
                dst.extend(vid * T + t for t in frames)
            start += n_sub
        out = torch.zeros(B * T, H, dtype=frame_sequence_output.dtype,
                          device=frame_sequence_output.device)
        if rows:
            dev = frame_sequence_output.device
            src = frame_sequence_output[torch.tensor(rows, device=dev),
                                        torch.tensor(ks, device=dev)]
            out.index_add_(0, torch.tensor(dst, device=dev), src)
        return out.view(B, T, H)

    def forward_vsm(self, batch):
        """model/model.py:226-237."""
        sub_query_batch = {"input_ids": batch["vsm_query_input_ids"],
                           "pos_ids": batch["vsm_query_pos_ids"],
                           "attn_masks": batch["vsm_query_attn_masks"]}
        return self.forward_repr_txt(batch, sub_query_batch)

    # ---- pretraining heads (model/model.py:239-336): encoder on CUDA, small heads in torch ----
    def forward_mfm(self, batch, compute_loss=True, loss="regression"):
        assert loss in ["regression", "nce"]
        if batch["f_v_feats"] is None:
            raise ValueError("MFM needs the batch's own f_v_feats: c_v_feats is overwritten in "
                             "place below and cannot also serve the subtitle-level frame slots")
        c_v_feats = batch["c_v_feats"]
        c_v_mask = batch["c_v_masks"]
        c_v_feats.masked_fill_(c_v_mask.unsqueeze(-1), 0)      # in place, like the reference
        batch["c_v_feats"] = c_v_feats + self.mask_embedding(c_v_mask.long())
        clip_outputs = self.forward_repr(batch)
        head_dtype = self.feat_regress.net[0].weight.dtype
        # masked / unmasked frame rows by index (their counts are host-known from the targets'
        # shape, so no boolean-mask compaction and no device->host read: model/model.py:249-257)
        flat_out = clip_outputs.reshape(-1, clip_outputs.size(-1))
        flat_mask = c_v_mask.reshape(-1)
        n_masked = batch["feat_targets"].shape[0] if batch["feat_targets"] is not None else None
        if n_masked is not None:
            idx = torch.nonzero_static(flat_mask, size=n_masked).reshape(-1)
        else:
            idx = torch.nonzero(flat_mask).reshape(-1)
        masked_output = flat_out[idx]
        prediction_feat = self.feat_regress(masked_output.to(head_dtype))
        neg_pred_feat = None
        if loss == "nce":
            if n_masked is not None:
                nidx = torch.nonzero_static(~flat_mask, size=flat_mask.numel() - n_masked).reshape(-1)
            else:
                nidx = torch.nonzero(~flat_mask).reshape(-1)
            neg_pred_feat = self.feat_regress(flat_out[nidx].to(head_dtype))
        if compute_loss:
            feat_targets = batch["feat_targets"]
            if loss == "regression":
                return F.mse_loss(prediction_feat, feat_targets, reduction="none")
            return self.mfm_nce(prediction_feat, feat_targets, neg_pred_feat)
        if loss == "regression":
            return prediction_feat
        return prediction_feat, neg_pred_feat

    def mfm_nce(self, masked_output, pos_output, neg_output, compute_loss=True):
        masked_score = masked_output.matmul(pos_output.t())
        neg_score = masked_output.matmul(neg_output.t())
        logits = torch.cat([masked_score, neg_score], dim=1).float()
        if compute_loss:
            targets = torch.arange(0, masked_output.size(0), dtype=torch.long,
                                   device=logits.device)
            return F.cross_entropy(logits / self.nce_temp, targets, reduction="none")
        return logits

    def forward_fom(self, batch, compute_loss=True):
        shuffled_orders = batch["shuffled_orders"]
        transformed = self.forward_repr(batch, encode_clip=False)
        expanded = shuffled_orders.unsqueeze(-1).expand_as(transformed)
        shuffled = torch.zeros_like(transformed).scatter_(1, expanded, transformed)
        encoded_clip = self.c_encoder(clip_level_pos_ids=None, clip_level_frame_feat=shuffled,
                                      attention_mask=batch["c_attn_masks"])
        bs, seq_len, hid = encoded_clip.size()
        out = self.fom_output(encoded_clip.view(bs * seq_len, hid).to(
            self.fom_output.linear_1.weight.dtype))
        if compute_loss:
            targets = batch["targets"].view(out.shape[0])
            return F.cross_entropy(out, targets, ignore_index=-1, reduction="mean")
        return out

    def initialize(self):
        self.apply(self.init_weights)
        self.f_encoder.apply(self.f_encoder.init_weights)
        self.c_encoder.apply(self.c_encoder.init_weights)

    def init_type_embedding(self):
        self.f_encoder.init_type_embedding()
        self.mask_embedding.weight.data[0].fill_(0)


class HeroModel(VideoPreTrainedModel):
    """model/model.py:348-364."""

    def __init__(self, config, vfeat_dim, max_frm_seq_len):
        super().__init__(config)
        self.config = config
        self.v_encoder = HierarchicalVlModel(config, vfeat_dim, max_frm_seq_len)
        self.v_encoder.initialize()

    def load_partial_pretrained(self, checkpoint, vfeat_dim, max_frm_seq_len, skip_layers=True):
        """RoBERTa-12 -> n-layer initialisation with the layer selection of
        model/modeling_utils.py:46-65: with gap = 12 // n_layers keep RoBERTa layers
        gap-1, 2*gap-1, ... and renumber them 0..n_layers-1."""
        n_layers = self.config.f_config.num_hidden_layers
        partial = dict(checkpoint)
        if skip_layers:
            gap = 12 // n_layers
            keep = {str(l): str(i) for i, l in enumerate(range(gap - 1, 12, gap))}
            partial = {}
            for k, v in checkpoint.items():
                if "roberta.encoder.layer." in k:
                    parts = k.split(".")
                    if parts[3] in keep:
                        parts[3] = keep[parts[3]]
                        partial[".".join(parts)] = v
                else:
                    partial[k] = v
        self.v_encoder.f_encoder = CrossModalTrm.from_pretrained(
            self.config.f_config, state_dict=partial, vfeat_dim=vfeat_dim,
            max_img_seq_len=max_frm_seq_len)
        self.v_encoder.f_encoder.pad_vocab()
        self.v_encoder.init_type_embedding()
        for m in (self, self.v_encoder):
            fp = m.__dict__.get("_hero_flat")
            if fp is not None:
                fp.invalidate()
