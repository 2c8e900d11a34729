"""Transformer layer modules with the reference's names, constructor arguments, parameter names
and shapes (model/layers.py), so checkpoints and the surrounding task heads keep working — but
`BertEncoder.forward` runs the hand-written packed CUDA pipeline instead of ~50 PyTorch ops/layer.

The per-op sub-modules (BertSelfAttention, BertIntermediate, ...) are parameter containers: their
arithmetic happens inside `functional.transformer_stack` (fused QKV GEMM, varlen attention, GEMM
epilogues with bias/GELU/dropout/residual, LayerNorm kernels).
"""
import torch
from torch import nn

from . import functional as Fn
from .params import flat_of
from .plan import TxtPlan

BF16 = torch.bfloat16


class BertLayerNorm(nn.LayerNorm):
    """Stands in for apex FusedLayerNorm (model/layers.py:8-9): same `weight`/`bias` names."""

    def __init__(self, hidden_size, eps=1e-12):
        super().__init__(hidden_size, eps=eps)


FusedLayerNorm = BertLayerNorm


class BertSelfAttention(nn.Module):
    """Parameters of model/layers.py:96-164 (query/key/value Linear + attention dropout)."""

    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError(
                "The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                % (config.hidden_size, config.num_attention_heads))
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = config.hidden_size // config.num_attention_heads
        self.all_head_size = self.num_attention_heads * self.attention_head_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(config.hidden_size, self.all_head_size)
        self.value = nn.Linear(config.hidden_size, self.all_head_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)

    def forward(self, input_tensor, attention_mask, head_mask=None):
        """Stand-alone use of one attention block on a padded batch (model/layers.py:124-179,
        182-231): the query-side `QueryFeatEncoder` runs it on 32 x 16 tokens, far off the hot
        path, so this is plain torch. `attention_mask` is the additive (N, 1, 1, L) mask of the
        reference. Returns a 1-tuple like the reference."""
        if head_mask is not None:
            raise ValueError("head_mask is not supported (always None in HERO)")
        sa = self.self
        N, L, _ = input_tensor.shape
        x = input_tensor.to(sa.query.weight.dtype)

        def heads(t):
            return t.view(N, L, sa.num_attention_heads, sa.attention_head_size).transpose(1, 2)

        q, k, v = heads(sa.query(x)), heads(sa.key(x)), heads(sa.value(x))
        scores = q @ k.transpose(-1, -2) / (sa.attention_head_size ** 0.5)
        probs = sa.dropout(torch.softmax(scores + attention_mask.to(scores.dtype), dim=-1))
        ctx = (probs @ v).transpose(1, 2).reshape(N, L, sa.all_head_size)
        out = self.output
        return (out.LayerNorm(out.dropout(out.dense(ctx)) + x),)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)
        if config.hidden_act != "gelu":
            raise ValueError("hero_b200 implements the erf-GELU of model/layers.py:16-25 only; "
                             f"got hidden_act={config.hidden_act!r}")


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class BertLayer(nn.Module):
    """model/layers.py:257-272."""

    def __init__(self, config):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)

    def ordered_params(self):
        a, i, o = self.attention, self.intermediate, self.output
        return [a.self.query.weight, a.self.query.bias, a.self.key.weight, a.self.key.bias,
                a.self.value.weight, a.self.value.bias, a.output.dense.weight,
                a.output.dense.bias, a.output.LayerNorm.weight, a.output.LayerNorm.bias,
                i.dense.weight, i.dense.bias, o.dense.weight, o.dense.bias, o.LayerNorm.weight,
                o.LayerNorm.bias]

    def weights(self, flat):
        """bf16 working views for the kernels; q/k/v are adjacent in the flat buffer."""
        a, i, o = self.attention, self.intermediate, self.output
        H = a.self.query.weight.shape[1]
        lw = Fn.LayerWeights()
        q, k, v = a.self.query, a.self.key, a.self.value
        if not (flat.contiguous_after(q.weight, k.weight) and
                flat.contiguous_after(k.weight, v.weight) and
                flat.contiguous_after(q.bias, k.bias) and flat.contiguous_after(k.bias, v.bias)):
            raise RuntimeError("query/key/value parameters are not adjacent in the flat buffer")
        lw.wqkv = flat.bf16_span(q.weight, 3 * H * H, (3 * H, H))
        lw.bqkv = flat.f32_span(q.bias, 3 * H, (3 * H,))
        lw.wo, lw.bo = flat.bf16(a.output.dense.weight), a.output.dense.bias
        lw.ln1_g, lw.ln1_b = a.output.LayerNorm.weight, a.output.LayerNorm.bias
        lw.w1, lw.b1 = flat.bf16(i.dense.weight), i.dense.bias
        lw.w2, lw.b2 = flat.bf16(o.dense.weight), o.dense.bias
        lw.ln2_g, lw.ln2_b = o.LayerNorm.weight, o.LayerNorm.bias
        return lw


class BertPooler(nn.Module):
    """model/layers.py:275-287. Dead on the encoder's 'repr' path (its output is discarded,
    model/model.py:196-198), so it stays a plain module evaluated only when a caller asks."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.activation = nn.Tanh()

    def forward(self, hidden_states):
        first = hidden_states[:, 0]
        return self.activation(self.dense(first.to(self.dense.weight.dtype)))


class BertEncoder(nn.Module):
    """model/layers.py:290-327: `forward(hidden_states (N, L, H), attention_mask (N, L) 0/1)`
    returns `(hidden,)`. `forward_packed` is the native entry used by the HERO encoders."""

    def __init__(self, config):
        super().__init__()
        self.output_attentions = getattr(config, "output_attentions", False)
        self.output_hidden_states = getattr(config, "output_hidden_states", False)
        if self.output_attentions or self.output_hidden_states:
            raise ValueError("hero_b200 does not materialise attention maps / per-layer states")
        self.num_heads = config.num_attention_heads
        self.eps = config.layer_norm_eps
        self.layer = nn.ModuleList([BertLayer(config) for _ in range(config.num_hidden_layers)])

    def dropout_state(self, base_key=None):
        if len(self.layer) == 0:
            return Fn.DropoutState()
        l0 = self.layer[0]
        return Fn.DropoutState(l0.output.dropout.p, l0.attention.self.dropout.p, self.training,
                               base_key)

    def forward_packed(self, x, att, drop=None, x_f32=None, out_f32=False):
        """x: packed bf16 [n_tokens, H]; att: device attention plan (`SeqPlan.attn`); x_f32: the
        same input in fp32 (residual of the first layer; derived from x when None); out_f32: return
        the last layer's fp32 output instead of its bf16 copy."""
        if len(self.layer) == 0:
            return x_f32 if (out_f32 and x_f32 is not None) else (x.float() if out_f32 else x)
        flat = flat_of(self, x.device)
        if drop is None:
            drop = self.dropout_state()
        # the per-layer views into the flat buffers and the parameter list only change when the
        # flat buffers are rebuilt: cache them (saves ~1 ms of Python per step over 9 layers)
        cache = self.__dict__.setdefault("_packed_cache", {})
        key = (flat.flat.data_ptr(), flat.mirror.data_ptr(), len(self.layer))
        if cache.get("key") != key:
            cache.clear()
            cache["key"] = key
            cache["layers"] = [l.weights(flat) for l in self.layer]
            cache["params"] = [p for l in self.layer for p in l.ordered_params()]
        params = cache["params"]
        cfg = {"layers": cache["layers"], "att": att, "heads": self.num_heads, "eps": self.eps,
               "drop": drop, "cache": cache, "out_f32": bool(out_f32)}
        cfg["flat"] = flat     # backward marks the bf16 mirror stale (an optimizer step follows)
        return Fn.transformer_stack(x, cfg, params, x_f32=x_f32)

    def forward(self, hidden_states, attention_mask=None, head_mask=None):
        if head_mask is not None:
            raise ValueError("head_mask is not supported (always None in HERO, layers.py:310)")
        N, L, H = hidden_states.shape
        if attention_mask is None:
            attention_mask = torch.ones(N, L, dtype=torch.long, device=hidden_states.device)
        plan = TxtPlan(attention_mask)
        dev = plan.to(hidden_states.device)
        flat_in = hidden_states.reshape(N * L, H)
        x32 = Fn.gather_rows(flat_in.float(), dev.f_tok_flat, dev.f_pad_to_tok)
        y = self.forward_packed(x32.to(BF16), plan.f.seq.attn(dev, "f_"), x_f32=x32.detach(),
                                out_f32=True)
        out = Fn.gather_rows(y, dev.f_pad_to_tok, dev.f_tok_flat)
        return (out.view(N, L, H).to(hidden_states.dtype),)


class LinearLayer(nn.Module):
    """model/layers.py:70-93 (LayerNorm -> Dropout -> Linear -> ReLU): parameter container for
    `frame_transform`; its arithmetic is fused into `functional.frame_merge`."""

    def __init__(self, in_hsz, out_hsz, layer_norm=True, dropout=0.1, relu=True):
        super().__init__()
        self.relu = relu
        self.layer_norm = layer_norm
        if layer_norm:
            self.LayerNorm = BertLayerNorm(in_hsz, eps=1e-5)
        self.net = nn.Sequential(nn.Dropout(dropout), nn.Linear(in_hsz, out_hsz))

    def forward(self, x):
        # Off the hot path (used by task heads on small inputs): plain torch.
        if self.layer_norm:
            x = self.LayerNorm(x)
        x = self.net(x)
        return torch.relu(x) if self.relu else x


def mask_logits(target, mask, eps=-1e4):
    """model/modeling_utils.py:42-43: keep `target` where mask == 1, `eps` elsewhere."""
    return target * mask + (1 - mask) * eps


def gelu(x):
    return x * 0.5 * (1.0 + torch.erf(x / 1.4142135623730951))


class GELU(nn.Module):
    def forward(self, input_):
        return gelu(input_)


class MLPLayer(nn.Module):
    """model/layers.py:48-61 (FOM head); off the encoder hot path, kept as torch ops."""

    def __init__(self, in_hsz, out_hsz):
        super().__init__()
        self.linear_1 = nn.Linear(in_hsz, in_hsz * 2)
        self.LayerNorm = BertLayerNorm(in_hsz * 2, eps=1e-5)
        self.linear_2 = nn.Linear(in_hsz * 2, out_hsz)

    def forward(self, x):
        return self.linear_2(self.LayerNorm(gelu(self.linear_1(x))))


class BertLMPredictionHead(nn.Module):
    """model/layers.py:330-354 (MLM head; 'next' row in SURVEY.md §8f): parameter-compatible
    torch module so CrossModalTrm.lm_head exists for checkpoints and the TVC decoder."""

    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-5)
        self.decoder = nn.Linear(bert_model_embedding_weights.size(1),
                                 bert_model_embedding_weights.size(0), bias=False)
        self.decoder.weight = bert_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(bert_model_embedding_weights.size(0)))

    def forward(self, hidden_states):
        h = self.LayerNorm(gelu(self.dense(hidden_states)))
        return self.decoder(h) + self.bias
