"""CPU oracle for the HERO hierarchical-encoder hot path.  TEST INFRASTRUCTURE ONLY.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this module. The product path (`hero_b200/`) never does and has no CPU fallback.

What this is: a functional fp32 restatement (plain torch ops on padded tensors, autograd for the
backward) of the arithmetic in the reference's
    model/layers.py   BertSelfAttention 124-164, BertSelfOutput 175-179, BertIntermediate 236-239 +
                      gelu 16-25, BertOutput 250-254, BertLayer 264-272, BertEncoder 298-327,
                      LinearLayer 86-93, BertPooler 281-287
    model/embed.py    SubEmbeddings 28-58, ImageEmbeddings 102-117, FrameEmbeddings 146-161
    model/encoder.py  CrossModalTrm._compute_img_txt_embeddings 256-285, forward_repr 336-352,
                      TemporalTrm.forward 404-423
    model/model.py    HierarchicalVlModel.collect_frame_outputs 156-187, forward_repr 195-224
    optim/adamw.py    AdamW.step 80-104
driven by the reference's own state_dict keys (so one set of weights feeds the reference, this
oracle and the CUDA path). It works on the PADDED layout with the additive -10000 mask exactly
like the reference, which makes it structurally independent of the packed CUDA implementation.

Pinning: the reference ships no golden vectors for this path (its only test is METEOR), so the
oracle is pinned against outputs of the unmodified reference modules imported in the build
container (`oracle/gen_golden.py` -> `tests/golden/*.npz`, checked by
`tests/test_oracle_golden.py`). apex FusedLayerNorm (not vendored; NGC 19.10 image) is restated as
standard LayerNorm: biased variance, fp32 statistics.
"""
import math

import torch


def layer_norm(x, weight, bias, eps):
    """apex FusedLayerNorm semantics (model/layers.py:8-9 import; standard LN over last dim)."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * weight + bias


def gelu_erf(x):
    """model/layers.py:16-25."""
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def linear(x, P, name):
    return x @ P[name + ".weight"].t() + P[name + ".bias"]


def bert_layer(h, add_mask, P, pfx, heads, eps, drop=None):
    """One BertLayer (model/layers.py:264-272). drop=None is eval mode (dropout = identity); else
    (probs [N, heads, L, L], attention-output [N, L, H], FFN-output [N, L, H]): scaled dropout
    masks (keep / (1 - p), or 0) multiplied in where the reference's nn.Dropout modules act —
    attention_probs (:149), BertSelfOutput (:177) and BertOutput (:252)."""
    N, L, H = h.shape
    m_probs, m_attn_out, m_ffn_out = (None, None, None) if drop is None else drop
    d = H // heads

    def split(t):  # transpose_for_scores, model/layers.py:118-122
        return t.view(N, L, heads, d).permute(0, 2, 1, 3)

    q = split(linear(h, P, pfx + "attention.self.query"))
    k = split(linear(h, P, pfx + "attention.self.key"))
    v = split(linear(h, P, pfx + "attention.self.value"))
    scores = q @ k.transpose(-1, -2) / math.sqrt(d) + add_mask      # :135-142
    probs = torch.softmax(scores, dim=-1)                           # :145
    if m_probs is not None:
        probs = probs * m_probs                                     # :149
    ctx = (probs @ v).permute(0, 2, 1, 3).reshape(N, L, H)          # :155-160
    o = linear(ctx, P, pfx + "attention.output.dense")
    if m_attn_out is not None:
        o = o * m_attn_out                                          # :177
    a = layer_norm(o + h,
                   P[pfx + "attention.output.LayerNorm.weight"],
                   P[pfx + "attention.output.LayerNorm.bias"], eps)  # :175-179
    f = gelu_erf(linear(a, P, pfx + "intermediate.dense"))          # :236-239
    o = linear(f, P, pfx + "output.dense")
    if m_ffn_out is not None:
        o = o * m_ffn_out                                           # :252
    return layer_norm(o + a,
                      P[pfx + "output.LayerNorm.weight"],
                      P[pfx + "output.LayerNorm.bias"], eps)         # :250-254


def bert_encoder(h, attn_mask, P, pfx, n_layers, heads, eps=1e-12):
    """BertEncoder.forward (model/layers.py:298-327): additive mask (1-m) * -10000."""
    add_mask = (1.0 - attn_mask[:, None, None, :].to(h.dtype)) * -10000.0
    for i in range(n_layers):
        h = bert_layer(h, add_mask, P, f"{pfx}layer.{i}.", heads, eps)
    return h


def sub_embeddings(P, pfx, input_ids, position_ids):
    """SubEmbeddings.forward (model/embed.py:28-58), token type fixed to 1 (:47-49)."""
    e = (P[pfx + "word_embeddings.weight"][input_ids]
         + P[pfx + "position_embeddings.weight"][position_ids]
         + P[pfx + "token_type_embeddings.weight"][1])
    return layer_norm(e, P[pfx + "LayerNorm.weight"], P[pfx + "LayerNorm.bias"], 1e-5)


def image_embeddings(P, pfx, type_row, img_feat, img_pos_ids, img_masks=None):
    """ImageEmbeddings.forward (model/embed.py:102-117)."""
    if img_masks is not None:
        img_feat = img_feat + P[pfx + "mask_embedding.weight"][img_masks.long()]
    x = layer_norm(img_feat, P[pfx + "img_LayerNorm.weight"], P[pfx + "img_LayerNorm.bias"], 1e-5)
    x = x @ P[pfx + "img_linear.weight"].t() + P[pfx + "img_linear.bias"]
    x = x + P[pfx + "position_embeddings.weight"][img_pos_ids] + type_row
    return layer_norm(x, P[pfx + "LayerNorm.weight"], P[pfx + "LayerNorm.bias"], 1e-5)


def cross_modal_embeddings(P, pfx, batch):
    """CrossModalTrm._compute_img_txt_embeddings (model/encoder.py:256-285)."""
    type_row = P[pfx + "embeddings.token_type_embeddings.weight"][1]
    txt = sub_embeddings(P, pfx + "embeddings.", batch["f_sub_input_ids"], batch["f_sub_pos_ids"])
    img = image_embeddings(P, pfx + "img_embeddings.", type_row, batch["f_v_feats"],
                           batch["f_v_pos_ids"], batch.get("f_v_masks"))
    cat = torch.cat([img, txt], dim=1)
    idx = batch["f_gather_index"].unsqueeze(-1).expand(-1, -1, cat.shape[-1])
    return torch.gather(cat, 1, idx)


def cross_modal_repr(P, pfx, batch, n_layers, heads):
    """CrossModalTrm.forward(batch, 'repr') -> sequence_output (model/encoder.py:297-311,336-352)."""
    emb = cross_modal_embeddings(P, pfx, batch)
    return bert_encoder(emb, batch["f_attn_masks"], P, pfx + "encoder.", n_layers, heads)


def cross_modal_txt(P, pfx, batch, n_layers, heads):
    """CrossModalTrm.forward(batch, 'txt') -> sequence_output (model/encoder.py:312-319)."""
    emb = sub_embeddings(P, pfx + "embeddings.", batch["input_ids"], batch["pos_ids"])
    return bert_encoder(emb, batch["attn_masks"], P, pfx + "encoder.", n_layers, heads)


def pooler(P, pfx, seq_out):
    """BertPooler (model/layers.py:281-287)."""
    return torch.tanh(seq_out[:, 0] @ P[pfx + "dense.weight"].t() + P[pfx + "dense.bias"])


def collect_frame_outputs(out_shape, frame_seq_out, num_subs, sub_idx2frame_idx):
    """HierarchicalVlModel.collect_frame_outputs (model/model.py:156-187), as one index_add."""
    B, T, H = out_shape
    rows, cols, dst = [], [], []
    start = 0
    for vid, n_sub in enumerate(num_subs):
        for sid, frames in sub_idx2frame_idx[vid]:
            for k, t in enumerate(frames):
                rows.append(start + sid)
                cols.append(k)
                dst.append(vid * T + t)
        start += n_sub
    out = torch.zeros(B * T, H, dtype=frame_seq_out.dtype)
    if rows:
        src = frame_seq_out[torch.tensor(rows), torch.tensor(cols)]
        out = out.index_add(0, torch.tensor(dst), src)
    return out.view(B, T, H)


def frame_transform(P, pfx, x):
    """LinearLayer.forward with layer_norm + relu (model/layers.py:86-93)."""
    x = layer_norm(x, P[pfx + "LayerNorm.weight"], P[pfx + "LayerNorm.bias"], 1e-5)
    return torch.relu(x @ P[pfx + "net.1.weight"].t() + P[pfx + "net.1.bias"])


def temporal_trm(P, pfx, frame_feat, attn_mask, n_layers, heads):
    """TemporalTrm.forward (model/encoder.py:404-423) with FrameEmbeddings (model/embed.py:146-161)."""
    T = frame_feat.shape[1]
    e = frame_feat + P[pfx + "embeddings.position_embeddings.weight"][torch.arange(T)][None]
    e = layer_norm(e, P[pfx + "embeddings.LayerNorm.weight"], P[pfx + "embeddings.LayerNorm.bias"],
                   1e-5)
    return bert_encoder(e, attn_mask, P, pfx + "encoder.", n_layers, heads)


def hierarchical_repr(P, batch, f_layers, c_layers, heads, encode_clip=True, pfx=""):
    """HierarchicalVlModel.forward_repr (model/model.py:195-224). P keys are relative to the
    HierarchicalVlModel (`f_encoder.*`, `frame_transform.*`, `c_encoder.*`), prefixed by pfx."""
    f_out = cross_modal_repr(P, pfx + "f_encoder.", batch, f_layers, heads)
    c_v = batch["c_v_feats"]
    shape = (c_v.shape[0], c_v.shape[1], f_out.shape[-1])
    matched = collect_frame_outputs(shape, f_out, batch["num_subs"], batch["sub_idx2frame_idx"])
    g = frame_transform(P, pfx + "frame_transform.", c_v) + matched
    if not encode_clip:
        return g
    return temporal_trm(P, pfx + "c_encoder.", g, batch["c_attn_masks"], c_layers, heads)


def adamw_step(p, g, m, v, step, lr, beta1, beta2, eps, weight_decay, correct_bias=True):
    """One AdamW update exactly as optim/adamw.py:80-104 (returns new p, m, v)."""
    m = m * beta1 + (1.0 - beta1) * g
    v = v * beta2 + (1.0 - beta2) * g * g
    denom = v.sqrt() + eps
    step_size = lr
    if correct_bias:
        step_size = lr * math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)
    p = p - step_size * (m / denom)
    if weight_decay > 0.0:
        p = p - lr * weight_decay * p
    return p, m, v


# ------------------------------------------------------------------ deterministic weights
def param_shapes(hidden=768, inter=3072, f_layers=6, c_layers=3, vocab=50272, max_pos=514,
                 type_vocab=2, vfeat_dim=4352, max_img_len=100):
    """state_dict keys/shapes of HierarchicalVlModel restricted to the encoder hot path
    (SURVEY.md §8b); key names are the reference's."""
    s = {}

    def layers(pfx, n):
        for i in range(n):
            b = f"{pfx}encoder.layer.{i}."
            for nm in ("query", "key", "value"):
                s[b + f"attention.self.{nm}.weight"] = (hidden, hidden)
                s[b + f"attention.self.{nm}.bias"] = (hidden,)
            s[b + "attention.output.dense.weight"] = (hidden, hidden)
            s[b + "attention.output.dense.bias"] = (hidden,)
            s[b + "attention.output.LayerNorm.weight"] = (hidden,)
            s[b + "attention.output.LayerNorm.bias"] = (hidden,)
            s[b + "intermediate.dense.weight"] = (inter, hidden)
            s[b + "intermediate.dense.bias"] = (inter,)
            s[b + "output.dense.weight"] = (hidden, inter)
            s[b + "output.dense.bias"] = (hidden,)
            s[b + "output.LayerNorm.weight"] = (hidden,)
            s[b + "output.LayerNorm.bias"] = (hidden,)

    f = "f_encoder."
    s[f + "embeddings.word_embeddings.weight"] = (vocab, hidden)
    s[f + "embeddings.position_embeddings.weight"] = (max_pos, hidden)
    s[f + "embeddings.token_type_embeddings.weight"] = (type_vocab, hidden)
    s[f + "embeddings.LayerNorm.weight"] = (hidden,)
    s[f + "embeddings.LayerNorm.bias"] = (hidden,)
    s[f + "img_embeddings.img_linear.weight"] = (hidden, vfeat_dim)
    s[f + "img_embeddings.img_linear.bias"] = (hidden,)
    s[f + "img_embeddings.img_LayerNorm.weight"] = (vfeat_dim,)
    s[f + "img_embeddings.img_LayerNorm.bias"] = (vfeat_dim,)
    s[f + "img_embeddings.position_embeddings.weight"] = (max_img_len, hidden)
    s[f + "img_embeddings.mask_embedding.weight"] = (2, vfeat_dim)
    s[f + "img_embeddings.LayerNorm.weight"] = (hidden,)
    s[f + "img_embeddings.LayerNorm.bias"] = (hidden,)
    s[f + "pooler.dense.weight"] = (hidden, hidden)
    s[f + "pooler.dense.bias"] = (hidden,)
    layers(f, f_layers)
    s["frame_transform.LayerNorm.weight"] = (vfeat_dim,)
    s["frame_transform.LayerNorm.bias"] = (vfeat_dim,)
    s["frame_transform.net.1.weight"] = (hidden, vfeat_dim)
    s["frame_transform.net.1.bias"] = (hidden,)
    c = "c_encoder."
    s[c + "embeddings.position_embeddings.weight"] = (max_pos, hidden)
    s[c + "embeddings.LayerNorm.weight"] = (hidden,)
    s[c + "embeddings.LayerNorm.bias"] = (hidden,)
    s[c + "pooler.dense.weight"] = (hidden, hidden)
    s[c + "pooler.dense.bias"] = (hidden,)
    layers(c, c_layers)
    return s


def seeded_weights(shapes, seed=0, std=0.02):
    """Deterministic weights independent of module construction order: one CPU generator walked
    over the keys in sorted order. LayerNorm gains ~1 +/- 0.1, biases ~N(0, std), matrices
    ~N(0, std) (the reference's initializer_range)."""
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        shp = shapes[k]
        t = torch.randn(*shp, generator=gen)
        if k.endswith("LayerNorm.weight"):
            t = 1.0 + 0.1 * t
        elif k.endswith("LayerNorm.bias") or k.endswith(".bias"):
            t = 0.05 * t
        else:
            t = std * t
        out[k] = t
    return out
