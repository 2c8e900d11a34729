"""CrossModalTrm / TemporalTrm with the reference's constructor + forward signatures
(model/encoder.py:204-423), running on the packed CUDA pipeline.

Differences in mechanism (not in results on valid positions):
  * embeddings are written straight into the packed `[frames, text]` token order by the fused
    gather+add+LayerNorm kernels — the cat + torch.gather of model/encoder.py:271-279 disappears;
  * padded positions are never computed; the padded outputs returned through the module API
    hold zeros there (the reference holds finite garbage that every caller masks out).
"""
import copy
import json
from collections import defaultdict

import torch
from torch import nn
from torch.nn import functional as F

from . import functional as Fn
from .embed import FrameEmbeddings, ImageEmbeddings, QueryFeatEmbeddings, SubEmbeddings
from .layers import (BertAttention, BertEncoder, BertLayerNorm, BertLMPredictionHead, BertPooler,
                     LinearLayer, gelu, mask_logits)
from .params import flat_of
from .plan import PLAN_KEY, TxtPlan, plan_inputs

BF16 = torch.bfloat16


class RobertaModelConfig(object):
    """Same fields/defaults as model/encoder.py:39-136 (layer_norm_eps defaults to 1e-12 because
    the HERO JSON configs omit it, model/encoder.py:54,110-117)."""

    def __init__(self, vocab_size_or_config_json_file, hidden_size=768, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                 hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                 max_position_embeddings=512, type_vocab_size=2, initializer_range=0.02,
                 layer_norm_eps=1e-12, **kwargs):
        if isinstance(vocab_size_or_config_json_file, str):
            with open(vocab_size_or_config_json_file, "r", encoding="utf-8") as reader:
                for key, value in json.loads(reader.read()).items():
                    self.__dict__[key] = value
        elif isinstance(vocab_size_or_config_json_file, int):
            self.vocab_size = vocab_size_or_config_json_file
            self.hidden_size = hidden_size
            self.num_hidden_layers = num_hidden_layers
            self.num_attention_heads = num_attention_heads
            self.hidden_act = hidden_act
            self.intermediate_size = intermediate_size
            self.hidden_dropout_prob = hidden_dropout_prob
            self.attention_probs_dropout_prob = attention_probs_dropout_prob
            self.max_position_embeddings = max_position_embeddings
            self.type_vocab_size = type_vocab_size
            self.initializer_range = initializer_range
            self.layer_norm_eps = layer_norm_eps
            self.output_attentions = kwargs.pop("output_attentions", False)
            self.output_hidden_states = kwargs.pop("output_hidden_states", False)
        else:
            raise ValueError("First argument must be either a vocabulary size (int) or the path "
                             "to a pretrained model config file (str)")

    @classmethod
    def from_dict(cls, json_object):
        config = RobertaModelConfig(vocab_size_or_config_json_file=-1)
        for key, value in json_object.items():
            config.__dict__[key] = value
        return config

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as reader:
            return cls.from_dict(json.loads(reader.read()))

    def to_dict(self):
        return copy.deepcopy(self.__dict__)

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"

    def __repr__(self):
        return str(self.to_json_string())


def load_pretrained_weight(model, state_dict):
    """Checkpoint loader with the reference's key conventions (model/modeling_utils.py:68-121):
    gamma/beta -> weight/bias, optional 'roberta.' prefix, missing/unexpected keys tolerated."""
    state_dict = dict(state_dict)
    for key in list(state_dict.keys()):
        new_key = key
        if "gamma" in new_key:
            new_key = new_key.replace("gamma", "weight")
        if "beta" in new_key:
            new_key = new_key.replace("beta", "bias")
        if new_key != key:
            state_dict[new_key] = state_dict.pop(key)
    if not hasattr(model, "roberta") and any(k.startswith("roberta.") for k in state_dict):
        state_dict = {k[len("roberta."):] if k.startswith("roberta.") else k: v
                      for k, v in state_dict.items()}
    own = model.state_dict()
    errors = []
    with torch.no_grad():
        for k, v in state_dict.items():
            if k in own:
                if own[k].shape != v.shape:
                    errors.append(f"size mismatch for {k}: {tuple(v.shape)} vs "
                                  f"{tuple(own[k].shape)}")
                else:
                    own[k].copy_(v)
    if errors:
        raise RuntimeError("Error(s) in loading state_dict for {}:\n\t{}".format(
            model.__class__.__name__, "\n\t".join(errors)))
    # the copies above went through state_dict views: tell the flat-parameter manager (if the
    # model has already run) that its bf16 working copy is stale
    for m in model.modules():
        fp = m.__dict__.get("_hero_flat")
        if fp is not None:
            fp.mark_dirty()
    return model


class RobertaPreTrainedModel(nn.Module):
    """model/encoder.py:139-201."""

    def __init__(self, config, *inputs, **kwargs):
        super().__init__()
        if not isinstance(config, RobertaModelConfig):
            raise ValueError(
                "Parameter config in `{}(config)` should be an instance of class "
                "`RobertaModelConfig`.".format(self.__class__.__name__))
        self.config = config

    def init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, BertLayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    @classmethod
    def load_config(cls, config):
        if isinstance(config, str):
            config = RobertaModelConfig.from_json_file(config)
        return config

    @classmethod
    def from_pretrained(cls, config_file, state_dict, *inputs, **kwargs):
        config = cls.load_config(config_file)
        model = cls(config, *inputs, **kwargs)
        return load_pretrained_weight(model, state_dict)


def _output_dtype(module):
    return getattr(module, "output_dtype", torch.float32)


class CrossModalTrm(RobertaPreTrainedModel):
    """Joint frame-subtitle encoder (model/encoder.py:204-389)."""

    def __init__(self, config, vfeat_dim, max_img_seq_len):
        super().__init__(config)
        self.encoder = BertEncoder(config)
        self.embeddings = SubEmbeddings(config)
        self.img_embeddings = ImageEmbeddings(config, vfeat_dim, max_img_seq_len)
        self.pooler = BertPooler(config)
        self.apply(self.init_weights)
        self.config = config
        self.lm_head = BertLMPredictionHead(config, self.embeddings.word_embeddings.weight)
        self.vocab_pad = 0
        self.register_buffer("pad", torch.zeros(8, config.hidden_size))
        self.output_dtype = torch.float32

    # ---- checkpoint helpers kept from the reference (model/encoder.py:226-235,287-295) ----
    def pad_vocab(self):
        emb_w = self.embeddings.word_embeddings.weight.data
        n_pad = (8 - emb_w.size(0) % 8) % 8
        if n_pad:
            emb_w = torch.cat([emb_w, emb_w.new_zeros(n_pad, emb_w.size(1))], 0)
            bias = torch.cat([self.lm_head.bias.data, self.lm_head.bias.data.new_zeros(n_pad)], 0)
        else:
            bias = self.lm_head.bias.data
        padded = nn.Parameter(emb_w)
        self.embeddings.word_embeddings.weight = padded
        self.lm_head.decoder.weight = padded
        self.lm_head.bias = nn.Parameter(bias)
        self.vocab_pad = n_pad
        self._invalidate_flat()

    def _invalidate_flat(self):
        fp = self.__dict__.get("_hero_flat")
        if fp is not None:
            fp.invalidate()

    def init_type_embedding(self):
        new_emb = nn.Embedding(2, self.config.hidden_size)
        new_emb.apply(self.init_weights)
        emb = self.embeddings.token_type_embeddings.weight.data[0, :]
        new_emb.weight.data[0, :].copy_(emb)
        new_emb.weight.data[1, :].copy_(emb)
        self.embeddings.token_type_embeddings = new_emb
        self._invalidate_flat()

    # ---- embedding API used by other heads (model/videoQA.py:73, model/violin.py:59) ----
    def _compute_txt_embeddings(self, input_ids, position_ids, txt_type_ids=None):
        return self.embeddings(input_ids=input_ids, position_ids=position_ids,
                               token_type_ids=txt_type_ids)

    # ---- packed hot path -------------------------------------------------------------------
    def _embed_cfg(self, fplan, dev, drop, img_feat, img_masks, shared_feats=None):
        """Arguments of functional.cross_modal_embed: the plan's index arrays (FPlan.embed_ids)
        and the frame features. `shared_feats`: clip-level frame features (B, T, D) to read the
        frame slots from when the batch carries no `f_v_feats` (plan.ReprPlan maps every packed
        frame token to its clip frame)."""
        cfg = {"drop": drop, "n_tok": fplan.n_tok, "n_txt": fplan.n_txt, "n_img": fplan.n_img,
               "pad_idx": self.embeddings.padding_idx, "img_mask": None}
        for k in ("txt_tok", "txt_ids", "txt_pos", "txtpos_off", "txtpos_idx", "img_tok",
                  "img_src", "img_pos", "imgpos_off", "imgpos_idx"):
            cfg[k] = getattr(dev, k)
        if fplan.n_img:
            if img_feat is None:
                if shared_feats is None:
                    raise ValueError("batch has neither f_v_feats nor c_v_feats for the frame slots")
                if img_masks is not None:
                    raise ValueError("frame masking (f_v_masks) needs the f_v_feats copy: the MFM "
                                     "path overwrites c_v_feats in place (model/model.py:244-247)")
                if not getattr(fplan, "shared_feats_ok", True):
                    raise ValueError("a frame slot marked valid in f_attn_masks is not listed in "
                                     "sub_idx2frame_idx: this batch cannot omit f_v_feats")
                img_feat, cfg["img_src"] = shared_feats, dev.img_src_c
            D = img_feat.shape[-1]
            feats = img_feat.reshape(-1, D)
            if feats.dtype != torch.float32:
                feats = feats.float()
            cfg["img_feats"] = feats.contiguous()
            if img_masks is not None:
                cfg["img_mask"] = img_masks.reshape(-1)[dev.img_src.long()].int()
        return cfg

    def _embed_params(self, with_img):
        e = self.embeddings
        params = [e.word_embeddings.weight, e.position_embeddings.weight,
                  e.token_type_embeddings.weight, e.LayerNorm.weight, e.LayerNorm.bias]
        if with_img:
            i = self.img_embeddings
            params += [i.img_linear.weight, i.img_linear.bias, i.img_LayerNorm.weight,
                       i.img_LayerNorm.bias, i.position_embeddings.weight,
                       i.mask_embedding.weight, i.LayerNorm.weight, i.LayerNorm.bias]
        return params

    def encode_packed(self, fplan, dev, att, img_feat=None, img_masks=None, drop=None,
                      shared_feats=None, out_f32=False):
        """Embeddings + encoder on the packed tokens of a plan (its FPlan, or a JointPlan) with
        device index `dev` and attention plan `att` -> [n_tokens, H], bf16 (feeds further
        kernels) or fp32 (`out_f32`: the caller unpacks it as the final result)."""
        flat = flat_of(self, dev.flat.device)
        if drop is None:
            drop = self.encoder.dropout_state()
        cfg = self._embed_cfg(fplan, dev, drop, img_feat, img_masks, shared_feats)
        with_img = fplan.n_img > 0
        if with_img:
            cfg["img_lin_w_bf16"] = flat.bf16(self.img_embeddings.img_linear.weight)
        emb, emb32 = Fn.cross_modal_embed(cfg, self._embed_params(with_img))
        return self.encoder.forward_packed(emb, att, drop, x_f32=emb32, out_f32=out_f32)

    def _unpack(self, y, dev, shape):
        out = Fn.gather_rows(y, dev.f_pad_to_tok, dev.f_tok_flat)
        out = out.view(shape[0], shape[1], y.shape[1])
        want = _output_dtype(self)
        return out if out.dtype == want else out.to(want)

    # ---- reference-facing API ---------------------------------------------------------------
    def forward(self, batch, task="repr", compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        if task == "repr":
            return self.forward_repr(batch["f_sub_input_ids"], batch["f_sub_pos_ids"],
                                     batch["f_v_feats"], batch["f_v_pos_ids"],
                                     batch["f_attn_masks"], batch["f_gather_index"],
                                     img_masks=batch["f_v_masks"], _plan=batch[PLAN_KEY])
        elif task == "txt":
            return self.forward_repr(input_ids=batch["input_ids"], position_ids=batch["pos_ids"],
                                     img_feat=None, img_pos_ids=None,
                                     attention_mask=batch["attn_masks"], gather_index=None,
                                     _plan=batch[PLAN_KEY])
        elif task.startswith("mlm"):
            return self.forward_mlm(batch["input_ids"], batch["position_ids"], batch["v_feat"],
                                    batch["f_pos_ids"], batch["attn_masks"],
                                    batch["gather_index"], batch["txt_mask_tgt"],
                                    batch["txt_labels"], compute_loss, _plan=batch[PLAN_KEY])
        else:
            raise ValueError(f"Unrecognized task {task}")

    def _plan_for(self, input_ids, position_ids, img_feat, img_pos_ids, attention_mask,
                  gather_index, _plan=None):
        """(FPlan, device index) of the attached plan, else of a TxtPlan built here (one
        device->host read of the masks and ids)."""
        if input_ids is None and img_feat is None:
            raise ValueError("Both img_feat and input_dis are None")
        if _plan is None:
            if input_ids is not None and img_feat is not None:
                assert gather_index is not None
            _plan = TxtPlan(**plan_inputs({
                "attn_masks": attention_mask, "input_ids": input_ids, "position_ids": position_ids,
                "gather_index": None if img_feat is None else gather_index,
                "f_pos_ids": None if img_feat is None else img_pos_ids, "v_feat": img_feat}, "mlm"))
        return _plan.f, _plan.to(attention_mask.device)

    def forward_repr(self, input_ids, position_ids, img_feat, img_pos_ids, attention_mask,
                     gather_index=None, txt_type_ids=None, img_type_ids=None, img_masks=None,
                     _plan=None):
        if txt_type_ids is not None or img_type_ids is not None:
            raise ValueError("explicit token type ids are not supported (HERO always uses 1)")
        fplan, dev = self._plan_for(input_ids, position_ids, img_feat, img_pos_ids,
                                    attention_mask, gather_index, _plan)
        y = self.encode_packed(fplan, dev, fplan.seq.attn(dev, "f_"), img_feat, img_masks,
                               out_f32=True)
        sequence_output = self._unpack(y, dev, attention_mask.shape)
        pooled_output = self.pooler(sequence_output)
        return (sequence_output, pooled_output)

    # ---- MLM (model/encoder.py:355-389); head stays torch ('next' row, SURVEY.md §8f) ------
    def mlm_head_input(self, input_ids, position_ids, img_feat, img_pos_ids, attention_mask,
                       gather_index, txt_mask_tgt, n_masked=None, _plan=None):
        """LM-head input h of the masked tokens (model/encoder.py:355-370): they are picked
        straight out of the PACKED encoder output (no padded tensor; with `n_masked`, the
        host-known number of masked tokens, no boolean-mask compaction either) and pass the
        LM-head transform (dense + gelu + LayerNorm, model/layers.py:336-346)."""
        fplan, dev = self._plan_for(input_ids, position_ids, img_feat, img_pos_ids,
                                    attention_mask, gather_index, _plan)
        y = self.encode_packed(fplan, dev, fplan.seq.attn(dev, "f_"), img_feat, out_f32=True)
        tgt = txt_mask_tgt.to(y.device, non_blocking=True).reshape(-1)
        if n_masked is not None:
            flat_idx = torch.nonzero_static(tgt, size=n_masked).reshape(-1)
        else:
            flat_idx = torch.nonzero(tgt).reshape(-1)
        tok = dev.f_pad_to_tok.long()[flat_idx]               # packed row of every masked token
        head = self.lm_head
        return head.LayerNorm(gelu(head.dense(y[tok].to(head.dense.weight.dtype))))

    def forward_mlm(self, input_ids, position_ids, img_feat, img_pos_ids, attention_mask,
                    gather_index, txt_mask_tgt, txt_labels=None, compute_loss=True, _plan=None):
        """model/encoder.py:355-374: `mlm_head_input`, then — when the loss is wanted — the fused
        vocabulary GEMM + cross entropy (functional.lm_head_cross_entropy): no (n_masked, 50272)
        logits tensor exists."""
        h = self.mlm_head_input(input_ids, position_ids, img_feat, img_pos_ids, attention_mask,
                                gather_index, txt_mask_tgt,
                                None if txt_labels is None else int(txt_labels.shape[0]), _plan)
        head = self.lm_head
        if compute_loss:
            flat = flat_of(self, h.device)
            emb = self.embeddings.word_embeddings.weight
            cfg = {"labels": txt_labels, "n_valid": emb.shape[0] - self.vocab_pad,
                   "emb_bf16": flat.bf16(emb)}
            return Fn.lm_head_cross_entropy(h, emb, head.bias, cfg)
        prediction_scores = head.decoder(h) + head.bias       # the caller asked for the logits
        if self.vocab_pad:
            prediction_scores = prediction_scores[:, :-self.vocab_pad]
        return prediction_scores


class TemporalTrm(RobertaPreTrainedModel):
    """Cross-frame encoder over the clip timeline (model/encoder.py:392-423)."""

    def __init__(self, config):
        super().__init__(config)
        self.embeddings = FrameEmbeddings(config)
        self.encoder = BertEncoder(config)
        self.pooler = BertPooler(config)
        self.apply(self.init_weights)
        self.output_dtype = torch.float32

    def embed_encode_packed(self, g, dev_t, att, pos_off, pos_idx, drop=None):
        """g: packed bf16 [n_c_tokens, H] -> FrameEmbeddings -> encoder -> packed FP32 output (the
        temporal transformer's output is the final result of the path)."""
        if drop is None:
            drop = self.encoder.dropout_state()
        e = self.embeddings
        cfg = {"drop": drop, "t": dev_t, "pos_off": pos_off, "pos_idx": pos_idx}
        z, z32 = Fn.frame_embed(g, cfg, [e.position_embeddings.weight, e.LayerNorm.weight,
                                         e.LayerNorm.bias])
        return self.encoder.forward_packed(z, att, drop, x_f32=z32, out_f32=True)

    def forward_encoder(self, embedding_output, attention_mask, pool=False):
        sequence_output = self.encoder(embedding_output, attention_mask)[0]
        if pool:
            return self.pooler(sequence_output)
        return sequence_output

    def forward(self, clip_level_frame_feat, clip_level_pos_ids, attention_mask):
        from .plan import SeqPlan, DeviceIndex, table_csr
        B, T, H = clip_level_frame_feat.shape
        sp = SeqPlan(attention_mask)
        arrays = sp.arrays("c_")
        if clip_level_pos_ids is None:
            t = sp.tok_col
        else:
            import numpy as np
            pid = clip_level_pos_ids.detach().cpu().numpy()
            pid = np.broadcast_to(pid, (B, T))
            t = pid[sp.tok_row, sp.tok_col].astype("int32")
        arrays["c_t"] = t
        arrays["c_pos_off"], arrays["c_pos_idx"] = table_csr(
            t, self.embeddings.position_embeddings.num_embeddings)
        dev = DeviceIndex(arrays, clip_level_frame_feat.device)
        flat_in = clip_level_frame_feat.reshape(B * T, H).to(BF16)
        g = Fn.gather_rows(flat_in, dev.c_tok_flat, dev.c_pad_to_tok)
        y = self.embed_encode_packed(g, dev.c_t, sp.attn(dev, "c_"), dev.c_pos_off,
                                     dev.c_pos_idx)
        out = Fn.gather_rows(y, dev.c_pad_to_tok, dev.c_tok_flat).view(B, T, H)
        want = _output_dtype(self)
        return out if out.dtype == want else out.to(want)


class QueryFeatEncoder(nn.Module):
    """model/encoder.py:426-485: projects query token features, adds positions, one self-attention
    block, and pools the tokens into ONE vector per query with a learned softmax over positions
    ("modularized query"). A 'next' row of SURVEY.md 8f: 32 queries x 16 tokens per step, plain
    torch on whatever device the features live on; parameter names match the reference."""

    def __init__(self, config, qfeat_dim, modularized=True):
        super().__init__()
        self.query_input_proj = LinearLayer(qfeat_dim, config.hidden_size, layer_norm=True,
                                            dropout=config.hidden_dropout_prob, relu=True)
        self.query_pos_embed = QueryFeatEmbeddings(config)
        self.query_self_attention = BertAttention(config)
        self.modularized = modularized
        if modularized:
            self.modular_vector_mapping = nn.Linear(config.hidden_size, 1, bias=False)

    def get_modularized_queries(self, query, query_mask, return_modular_att=False):
        """query (N, L, D), query_mask (N, L) -> (N, D): softmax over the valid positions of a
        learned per-token score, used as pooling weights."""
        scores = self.modular_vector_mapping(query)                       # (N, L, 1)
        att = torch.softmax(mask_logits(scores, query_mask.unsqueeze(2)), dim=1)
        pooled = (att * query).sum(1)                                      # (N, D)
        return (pooled, att) if return_modular_att else pooled

    def forward(self, query_feat, query_attn_mask, query_pos_ids=None):
        dtype = next(self.parameters()).dtype
        x = self.query_pos_embed(self.query_input_proj(query_feat.to(dtype)))
        mask = query_attn_mask.to(dtype)
        attended = self.query_self_attention(x, (1.0 - mask)[:, None, None, :] * -10000.0)[0]
        return self.get_modularized_queries(attended, mask) if self.modularized else attended
