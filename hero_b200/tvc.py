"""HeroForTvc and TvcGenerator (model/tvc.py): TVC video captioning, inference.

The encoder is HERO's ('repr'); each caption segment is a frame range of its video's clip-level
output. The decoder is a 2-layer transformer with causal self-attention and cross-attention to the
segment frames, its word embedding and LM head tied to the cross-modal encoder's. On this path:

    ReprPlan + TvcPlan (host)  ->  repr_packed  ->  gather the segment rows (+ one zero row)  ->
    per decoder layer: cross K / V of all segment frames, one GEMM
    per position: word[id] + pos[t] -> LayerNorm (ln_fwd) -> per layer: QKV GEMM, dec_attn_fwd
      (causal range), dense + residual -> LayerNorm, Q GEMM, dec_attn_fwd (segment range),
      dense + residual -> LayerNorm, FFN (GELU) -> dense + residual -> LayerNorm  ->
    LM-head transform (GEMM + GELU, LayerNorm) -> vocabulary GEMM (fp32 logits)

`forward` runs that over every position of the teacher-forced captions at once. Greedy decoding
runs it one position at a time against a KV cache that the QKV GEMM writes straight into, and takes
the argmax with `rank_topk(k=1)` into the next step's id buffer: the reference instead re-runs the
decoder and the full-vocabulary logits over the whole prefix at every step (model/tvc.py:301-330).
Beam search runs the same pass over n_captions x beam rows: `beam_logprob_topk` gives each row's
log-probabilities' top-B in one read of its logits, `beam_select` picks each caption's next beams
on the device, and self-attention gathers each beam's keys through its KV-ancestry table
(`dec_attn_gather_fwd`), so reordering beams copies no cache. Sampling runs greedy decoding's loop
with `sample_tokens` (temperature, top-k, top-p and a Gumbel-max draw keyed by (seed, row, step))
in place of the argmax, and the decoding controls (no_repeat_ngram_size, min_length) write -inf
into each step's logits with `ban_tokens` before any of the three selections. With `early_stop`,
`dec_finished` records on the device the first step at which every row has ended and mirrors it
into a pinned host word; the host reads that word with a plain load before it enqueues each step
and stops enqueueing once it is set, so the loop still never synchronises.

Inference only. Decoder training (its attention backward and the label-smoothed loss gradient) is
not on the CUDA path yet: `forward` raises NotImplementedError in training mode or when it would
have to build an autograd graph.
"""
import math
from collections import defaultdict

import numpy as np
import torch
from torch import nn

from . import ops
from .layers import BertIntermediate, BertLayerNorm, BertOutput, BertSelfAttention, BertSelfOutput
from .model import HeroModel
from .params import flat_of
from .plan import PLAN_KEY, ReprPlan, TvcPlan, plan_inputs

BF16 = torch.bfloat16
MAX_DECODE_STEP = 1023      # position table of 1024 entries (hero_tvc.json d_config)


class LabelSmoothingLoss(nn.Module):
    """Parameter container of model/tvc.py:19-64 (its `one_hot` buffer is part of the reference's
    state_dict). The loss itself is computed from the fused LM-head cross entropy in
    `HeroForTvc._loss`."""

    def __init__(self, label_smoothing, tgt_vocab_size, ignore_index=-100, reduction="none"):
        assert 0.0 < label_smoothing <= 1.0
        super().__init__()
        self.ignore_index = ignore_index
        self.smoothing_value = label_smoothing / (tgt_vocab_size - 1)
        self.register_buffer("one_hot", torch.full((tgt_vocab_size,),
                                                   self.smoothing_value).unsqueeze(0))
        self.confidence = 1.0 - label_smoothing
        self.reduction = reduction


class BertDecoderLayer(nn.Module):
    """model/tvc.py:107-154 (parameter names kept, `intermidiate` included)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.self_attention = BertSelfAttention(config)
        self.add_norm_1 = BertSelfOutput(config)
        self.dec_enc_attention = BertSelfAttention(config)
        self.add_norm_2 = BertSelfOutput(config)
        self.intermidiate = BertIntermediate(config)
        self.add_norm_3 = BertOutput(config)

    def weights(self, flat):
        """bf16 GEMM operands and fp32 biases / LayerNorm parameters of the layer; q / k / v of
        both attentions are adjacent in the flat buffer (params._ordered_named_params)."""
        sa, ca = self.self_attention, self.dec_enc_attention
        H = sa.query.weight.shape[1]
        for a, b in ((sa.query, sa.key), (sa.key, sa.value), (ca.key, ca.value)):
            if not (flat.contiguous_after(a.weight, b.weight) and
                    flat.contiguous_after(a.bias, b.bias)):
                raise RuntimeError("decoder query/key/value parameters are not adjacent in the "
                                   "flat buffer")
        n1, n2, n3 = self.add_norm_1, self.add_norm_2, self.add_norm_3
        return {
            "wqkv": flat.bf16_span(sa.query.weight, 3 * H * H, (3 * H, H)),
            "bqkv": flat.f32_span(sa.query.bias, 3 * H, (3 * H,)),
            "wo1": flat.bf16(n1.dense.weight), "bo1": n1.dense.bias.detach(), "ln1": n1.LayerNorm,
            "wq_c": flat.bf16(ca.query.weight), "bq_c": ca.query.bias.detach(),
            "wkv_c": flat.bf16_span(ca.key.weight, 2 * H * H, (2 * H, H)),
            "bkv_c": flat.f32_span(ca.key.bias, 2 * H, (2 * H,)),
            "wo2": flat.bf16(n2.dense.weight), "bo2": n2.dense.bias.detach(), "ln2": n2.LayerNorm,
            "w1": flat.bf16(self.intermidiate.dense.weight),
            "b1": self.intermidiate.dense.bias.detach(),
            "w2": flat.bf16(n3.dense.weight), "b2": n3.dense.bias.detach(), "ln3": n3.LayerNorm,
        }


class BertDecoder(nn.Module):
    """model/tvc.py:157-193: the layers and the persistent causal-mask buffer of the reference
    (kept for its state_dict; the kernels take key ranges instead)."""

    def __init__(self, config):
        super().__init__()
        self.num_heads = config.num_attention_heads
        self.layer = nn.ModuleList([BertDecoderLayer(config)
                                    for _ in range(config.num_hidden_layers)])
        tri_mask = torch.tril(torch.ones(1024, 1024), diagonal=0)
        tri_mask = (1.0 - tri_mask) * -10000.0
        self.register_buffer("tri_mask", tri_mask)


def _ln(x, ln, y, n_rows, y_f32=None, **kw):
    ops.ln_fwd(x, ln.weight.detach(), ln.bias.detach(), ln.eps, y, n_rows=n_rows, y_f32=y_f32,
               **kw)


class _Workspace:
    """Activation buffers of one decoder pass over m rows (reused by every layer / step)."""

    def __init__(self, m, H, inter, V, device):
        f32 = torch.float32
        self.x, self.a, self.b = (torch.empty(m, H, dtype=BF16, device=device) for _ in range(3))
        self.x32, self.a32, self.b32 = (torch.empty(m, H, dtype=f32, device=device)
                                        for _ in range(3))
        self.s = torch.empty(m, H, dtype=f32, device=device)
        self.ctx = torch.empty(m, H, dtype=BF16, device=device)
        self.qc = torch.empty(m, H, dtype=BF16, device=device)
        self.f = torch.empty(m, inter, dtype=BF16, device=device)
        self.t = torch.empty(m, H, dtype=BF16, device=device)
        self.h = torch.empty(m, H, dtype=BF16, device=device)
        self.logits = torch.empty(m, V, dtype=f32, device=device)


class HeroForTvc(HeroModel):
    def __init__(self, config, vfeat_dim, max_frm_seq_len, lsr=0.1):
        super().__init__(config, vfeat_dim, max_frm_seq_len)
        self.config = config
        d = config.d_config
        self.position_embeddings = nn.Embedding(d.max_position_embeddings, d.hidden_size)
        self.emb_LayerNorm = BertLayerNorm(d.hidden_size, eps=1e-5)
        self.decoder = BertDecoder(d)
        self.lsr = lsr
        if lsr > 0:
            self.loss_func = LabelSmoothingLoss(lsr, config.f_config.vocab_size, ignore_index=-1,
                                                reduction="none")
        else:
            self.loss_func = nn.CrossEntropyLoss(ignore_index=-1, reduction="none")
        self.v_encoder.initialize()

    # ------------------------------------------------------------------ encoder side
    def encode(self, batch):
        """model/tvc.py:219-238 without the padding: (packed clip-level outputs fp32
        [n_c_tokens, H] of HierarchicalVlModel.repr_packed, TvcPlan of the caption segments). Uses
        the ReprPlan attached with plan.attach_plan, else builds it (one device->host read of the
        masks and ids)."""
        if not isinstance(batch, defaultdict):
            batch = defaultdict(lambda: None, batch)
        rplan = batch[PLAN_KEY]
        if rplan is None:
            rplan = ReprPlan(plan_inputs(batch))
        tplan = TvcPlan(batch["clip_ranges"], rplan)
        flat_of(self, batch["c_v_feats"].device)   # one flat buffer for encoder and decoder
        y, _ = self.v_encoder.repr_packed(batch, rplan)
        return y, tplan

    def _gather_segments(self, y, tplan, tdev):
        rows = torch.empty(tplan.n_rows, y.shape[1], dtype=y.dtype, device=y.device)
        ops.gather_rows(y.contiguous(), tdev.seg_src, rows)
        if rows.dtype == BF16:
            return rows
        return ops.cast_bf16(rows, torch.empty(rows.shape, dtype=BF16, device=y.device))

    def _weights(self, device):
        flat = flat_of(self, device)
        fe = self.v_encoder.f_encoder
        head = fe.lm_head
        emb = fe.embeddings.word_embeddings.weight
        return flat, {
            "layers": [l.weights(flat) for l in self.decoder.layer],
            "word": emb.detach(), "pos": self.position_embeddings.weight.detach(),
            "emb_bf16": flat.bf16(emb), "lm_bias": head.bias.detach(),
            "dense": flat.bf16(head.dense.weight), "dense_b": head.dense.bias.detach(),
            "n_valid": emb.shape[0] - fe.vocab_pad}

    def _cross_kv(self, w, enc):
        """Cross-attention K | V [rows + 1, 2H] of every decoder layer, one GEMM each."""
        out = []
        for lw in w["layers"]:
            kv = torch.empty(enc.shape[0], lw["wkv_c"].shape[0], dtype=BF16, device=enc.device)
            out.append(ops.gemm(enc, lw["wkv_c"], kv, bias=lw["bkv_c"]))
        return out

    def _check_inference(self):
        if self.training or (torch.is_grad_enabled() and
                             any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError(
                "TVC decoder training is not on the CUDA path yet: HeroForTvc runs inference "
                "only. Call it in eval mode under torch.no_grad().")

    # ------------------------------------------------------------------ decoder
    def _self_attn_range(self, off, ln, max_len):
        """Self-attention of a pass whose keys are the ranges [off[i], off[i] + ln[i])."""
        heads = self.decoder.num_heads
        return lambda q, k, v, out: ops.dec_attn_fwd(q, k, v, off, ln, out, heads=heads,
                                                     max_kv_len=max_len)

    def _self_attn_gather(self, kv_idx, ln, max_len):
        """Self-attention of a pass whose key j of row i is cache row kv_idx[i, j], j < ln[i]."""
        heads = self.decoder.num_heads
        return lambda q, k, v, out: ops.dec_attn_gather_fwd(q, k, v, kv_idx, ln, out, heads=heads,
                                                            max_kv_len=max_len)

    def _positions(self, w, ws, ids, pos, n_rows, layers, self_qkv, self_attn, cross_kv, cross_rng):
        """One decoder pass over n_rows positions: embedding, every layer, LM-head transform and
        the vocabulary logits (into ws.logits). `self_qkv(l)` -> (QKV output view, K view, V view)
        of layer l; `self_attn(q, k, v, out)` launches the self-attention (_self_attn_range /
        _self_attn_gather); `cross_rng` = (kv_off, kv_len, max_len)."""
        H = ws.x.shape[1]
        heads = self.decoder.num_heads
        _ln(w["word"], self.emb_LayerNorm, ws.x, n_rows, y_f32=ws.x32, x_rows=ids,
            add_tab=w["pos"], add_idx=pos)
        for l, lw in enumerate(layers):
            qkv, k, v = self_qkv(l)
            ops.gemm(ws.x, lw["wqkv"], qkv, bias=lw["bqkv"])
            self_attn(qkv[:, :H], k, v, ws.ctx)
            ops.gemm(ws.ctx, lw["wo1"], ws.s, bias=lw["bo1"], resid=ws.x32)
            _ln(ws.s, lw["ln1"], ws.a, n_rows, y_f32=ws.a32)
            ops.gemm(ws.a, lw["wq_c"], ws.qc, bias=lw["bq_c"])
            kv = cross_kv[l]
            ops.dec_attn_fwd(ws.qc, kv[:, :H], kv[:, H:], cross_rng[0], cross_rng[1], ws.ctx,
                             heads=heads, max_kv_len=cross_rng[2])
            ops.gemm(ws.ctx, lw["wo2"], ws.s, bias=lw["bo2"], resid=ws.a32)
            _ln(ws.s, lw["ln2"], ws.b, n_rows, y_f32=ws.b32)
            ops.gemm(ws.b, lw["w1"], ws.f, bias=lw["b1"], act=ops.ACT_GELU)
            ops.gemm(ws.f, lw["w2"], ws.s, bias=lw["b2"], resid=ws.b32)
            _ln(ws.s, lw["ln3"], ws.x, n_rows, y_f32=ws.x32)
        head = self.v_encoder.f_encoder.lm_head
        ops.gemm(ws.x, w["dense"], ws.t, bias=w["dense_b"], act=ops.ACT_GELU)
        _ln(ws.t, head.LayerNorm, ws.h, n_rows)
        ops.gemm(ws.h, w["emb_bf16"], ws.logits, bias=w["lm_bias"])

    def _workspace(self, m, device):
        d = self.config.d_config
        V = self.v_encoder.f_encoder.embeddings.word_embeddings.weight.shape[0]
        return _Workspace(m, d.hidden_size, d.intermediate_size, V, device)

    def forward(self, batch, mode="train", compute_loss=True):
        """model/tvc.py:268-276. Without `compute_loss`: the teacher-forced logits (N, Lt, V) fp32,
        every position computed (padded ones included). With it: the reference's per-token loss,
        LabelSmoothingLoss over the positions whose target is not -1 (lsr > 0), or cross entropy
        with ignore_index -1 over all N * Lt positions (lsr == 0)."""
        self._check_inference()
        ids = batch["cap_input_ids"]
        N, Lt = ids.shape
        if Lt > self.position_embeddings.num_embeddings:
            raise ValueError(f"captions of {Lt} tokens exceed the position table")
        y, tplan = self.encode(batch)
        device = y.device
        if tplan.n_seg != N:
            raise ValueError(f"{N} captions but {tplan.n_seg} segments in clip_ranges")
        tdev = tplan.to(device, tplan.forced_arrays(Lt))
        enc = self._gather_segments(y, tplan, tdev)
        flat, w = self._weights(device)
        cross = self._cross_kv(w, enc)
        M = N * Lt
        ws = self._workspace(M, device)
        H = ws.x.shape[1]
        qkv = torch.empty(M, 3 * H, dtype=BF16, device=device)
        pos = batch["cap_pos_ids"].to(device=device)
        pos = pos.expand(N, Lt).reshape(-1).to(torch.int32)
        self._positions(w, ws, ids.to(device=device).reshape(-1).to(torch.int32), pos, M,
                        w["layers"], lambda l: (qkv, qkv[:, H:2 * H], qkv[:, 2 * H:]),
                        self._self_attn_range(tdev.tf_self_off, tdev.tf_self_len, Lt),
                        cross, (tdev.tf_kv_off, tdev.tf_kv_len, tplan.max_kv))
        n_valid = w["n_valid"]
        if not compute_loss:
            return ws.logits[:, :n_valid].view(N, Lt, n_valid)
        return self._loss(ws, w, batch["cap_tgt_ids"], n_valid)

    def _loss(self, ws, w, tgt, V):
        device = ws.h.device
        labels = tgt.reshape(-1).to(device)
        valid = labels != -1
        lab32 = torch.where(valid, labels, torch.zeros_like(labels)).to(torch.int32)
        ce, lse = ops.lm_head_ce_fwd(ws.h, w["emb_bf16"], w["lm_bias"], lab32, V)
        if self.lsr <= 0:
            return torch.where(valid, ce, torch.zeros_like(ce))
        # KL(q || softmax(z)) summed over the V columns, q = conf at the target, s elsewhere:
        #   sum q log q - conf (z_t - lse) - s (sum_j z_j - z_t - (V - 1) lse)
        # with z_t = lse - ce and sum_j z_j = h . sum_j E_j + sum_j b_j (one mat-vec against the
        # column sum of the tied table)
        lf = self.loss_func
        conf, s = lf.confidence, lf.smoothing_value
        esum = torch.zeros(ws.h.shape[1], dtype=torch.float32, device=device)
        ops.colsum(w["emb_bf16"][:V], esum)
        e8 = torch.zeros(8, ws.h.shape[1], dtype=BF16, device=device)
        ops.cast_bf16(esum, e8[0])
        zs8 = torch.empty(ws.h.shape[0], 8, dtype=torch.float32, device=device)
        ops.gemm(ws.h, e8, zs8)
        zsum = zs8[:, 0] + w["lm_bias"][:V].sum()
        zt = lse - ce
        ent = conf * math.log(conf) + (V - 1) * s * math.log(s)
        loss = ent - conf * (zt - lse) - s * (zsum - zt - (V - 1) * lse)
        if tgt.device.type == "cpu":
            keep = torch.from_numpy(np.flatnonzero(tgt.reshape(-1).numpy() != -1)).to(device)
            return loss[keep]
        return loss[valid]


class TvcGenerator(object):
    """model/tvc.py:293-338 with the reference's constructor. `fp16` is accepted and ignored: the
    path runs in bf16. `greedy_decode(batch)` returns, per caption, the greedy ids cut at the first
    EOS, like the reference; it runs `max_step` positions (fewer with `early_stop`) with a KV cache
    and returns the token chosen at each step, where the reference re-derives every position
    from its last full pass (equal under causal masking). `beam_search(batch, beam_size,
    length_penalty)` decodes with a beam and `sample(batch, ...)` draws one caption per segment, on
    the same path (neither is in the reference).

    Decoding controls, applied by every method to the logits of each step before the selection
    (`ops.ban_tokens`; 0 turns a control off, and with both off no kernel runs for them):
    `no_repeat_ngram_size` n bans every token that would complete an n-gram already present in
    [bos] + the row's history, and `min_length` bans EOS at the steps t < min_length. A banned
    token gets logit -inf, so its probability is 0 and the others are renormalised (beam scores
    included).

    `early_stop` (off by default) stops enqueueing steps once every row has ended: the first step
    after whose selection every caption (every beam of every caption, in beam search) has emitted
    EOS is recorded on the device (`ops.dec_finished`) and read by the host from pinned memory
    without a synchronisation. Steps the host enqueued before it saw the word still run; every
    position after the recorded step is then filled with EOS, so the output does not depend on how
    far ahead of the device the host was. Greedy and sampled ids equal the full run's up to and
    including that step and are EOS after it (the captions, cut at the first EOS, are the same);
    beam_ids is bitwise the full run's."""

    def __init__(self, model, max_step, bos, eos, fp16, *, min_length=0, no_repeat_ngram_size=0,
                 early_stop=False):
        if not isinstance(early_stop, bool):
            raise ValueError(f"early_stop = {early_stop!r}: must be True or False")
        self.model = model
        self.max_step = max_step
        self.bos = bos
        self.eos = eos
        self.fp16 = fp16
        self.min_length = min_length
        self.no_repeat_ngram_size = no_repeat_ngram_size
        self.early_stop = early_stop

    def _n_valid(self):
        fe = self.model.v_encoder.f_encoder
        return fe.embeddings.word_embeddings.weight.shape[0] - fe.vocab_pad

    def _check_controls(self, n_valid):
        """The controls' bounds: at most max_step n-gram bans and EOS fall on one row, so
        max_step + 2 columns guarantee that a row is never fully masked."""
        n, m = self.no_repeat_ngram_size, self.min_length
        if int(n) != n or n < 0:
            raise ValueError(f"no_repeat_ngram_size = {n}: must be an integer >= 0")
        if int(m) != m or m < 0:
            raise ValueError(f"min_length = {m}: must be an integer >= 0")
        if (n or m) and int(self.max_step) + 2 > n_valid:
            raise ValueError(f"max_step = {self.max_step}: with no_repeat_ngram_size or min_length "
                             f"on, max_step + 2 must not exceed the {n_valid} vocabulary entries")

    def _ban(self, logits, n_valid, hist, step_stride, row_stride, t):
        if self.no_repeat_ngram_size or self.min_length:
            ops.ban_tokens(logits, n_valid, hist, step_stride=step_stride, row_stride=row_stride,
                           bos=int(self.bos), step=t, ngram=int(self.no_repeat_ngram_size),
                           min_length=int(self.min_length), eos=int(self.eos))

    @torch.no_grad()
    def greedy_decode(self, batch):
        ids = self.decode_ids(batch)
        return [self.cut_eos(row) for row in ids.tolist()]

    @torch.no_grad()
    def decode_ids(self, batch):
        """Greedy ids (n_captions, max_step) as a host int32 tensor. Every upload of the batch
        happens before the loop; the ids come back in one device->host copy. With early_stop, the
        columns after the step at which every caption had emitted EOS are EOS."""
        return self._decode_rows(batch, "greedy decoding", None)

    @torch.no_grad()
    def sample(self, batch, *, temperature=1.0, top_k=0, top_p=1.0, seed=0):
        """Per caption, one sampled caption (see sample_ids), cut at the first EOS."""
        ids = self.sample_ids(batch, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed)
        return [self.cut_eos(row) for row in ids.tolist()]

    @torch.no_grad()
    def sample_ids(self, batch, *, temperature=1.0, top_k=0, top_p=1.0, seed=0):
        """Sampled ids (n_captions, max_step) as a host int32 tensor: greedy decoding's loop with
        `ops.sample_tokens` in place of the argmax. Each step divides the logits by `temperature`,
        keeps the columns at or above the `top_k`-th largest (0: all), then the smallest set of the
        largest columns whose probability reaches `top_p` (1: all), and draws from the
        renormalised distribution by Gumbel-max. The uniforms are a hash of (seed, caption row,
        step, column), so the same batch and seed give the same ids (csrc/decode_ctl.cu). One
        upload before the loop, one device->host copy after it."""
        if not (float(temperature) > 0.0 and math.isfinite(float(temperature))):
            raise ValueError(f"temperature = {temperature}: must be > 0")
        if int(top_k) != top_k or top_k < 0:
            raise ValueError(f"top_k = {top_k}: must be an integer >= 0 (0 keeps every token)")
        if not 0.0 < float(top_p) <= 1.0:
            raise ValueError(f"top_p = {top_p}: must lie in (0, 1] (1 keeps every token)")
        _check_seed(seed)
        if self._n_valid() > ops.SAMPLE_MAX_COLS:
            raise ValueError(f"{self._n_valid()} vocabulary entries: sampling takes at most "
                             f"{ops.SAMPLE_MAX_COLS}")
        return self._decode_rows(batch, "sampling", dict(
            temperature=float(temperature), top_k=int(top_k), top_p=float(top_p), seed=int(seed)))

    def _prepare(self, batch, what, arrays, per_caption=1, check=None):
        """Checks max_step (for strategy `what`), then `check(n_valid)`, the controls and inference
        mode; encodes the batch and uploads its plan arrays `arrays(tplan)`. Returns (tplan, tdev,
        weights, cross K / V, workspace of n_captions * per_caption rows)."""
        model, T = self.model, int(self.max_step)
        if not 1 <= T <= MAX_DECODE_STEP:
            raise ValueError(f"max_step = {T}: {what} takes 1 to {MAX_DECODE_STEP} steps "
                             f"(position table of {MAX_DECODE_STEP + 1})")
        n_valid = self._n_valid()
        if check is not None:
            check(n_valid)
        self._check_controls(n_valid)
        model._check_inference()
        y, tplan = model.encode(batch)
        device = y.device
        tdev = tplan.to(device, arrays(tplan))
        enc = model._gather_segments(y, tplan, tdev)
        _, w = model._weights(device)
        cross = model._cross_kv(w, enc)
        ws = model._workspace(tplan.n_seg * per_caption, device)
        return tplan, tdev, w, cross, ws

    def _decode_rows(self, batch, what, sampling):
        """The one-row-per-caption loop of greedy decoding and sampling: `sampling` None picks the
        argmax with rank_topk(k=1), else ops.sample_tokens with these keyword arguments."""
        model, T = self.model, int(self.max_step)
        tplan, tdev, w, cross, ws = self._prepare(batch, what, lambda p: p.decode_arrays(T))
        device, N, H = ws.x.device, tplan.n_seg, ws.x.shape[1]
        caches = [torch.empty(N, T, 3 * H, dtype=BF16, device=device) for _ in w["layers"]]
        rows = [c.view(N * T, 3 * H) for c in caches]
        out = torch.empty(T + 1, N, dtype=torch.int32, device=device)
        out[0].fill_(int(self.bos))
        vals = torch.empty(N, 1, dtype=torch.float32, device=device)
        n_valid = w["n_valid"]
        stop = _EarlyStop(device, int(self.eos), N) if self.early_stop else None
        for t in range(T):
            if stop is not None and t and stop.reached():
                break
            step = slice(t * N, (t + 1) * N)
            model._positions(w, ws, out[t], tdev.step_pos[step], N, w["layers"],
                             lambda l: (caches[l][:, t], rows[l][:, H:2 * H], rows[l][:, 2 * H:]),
                             model._self_attn_range(tdev.self_off, tdev.step_len[step], t + 1),
                             cross, (tdev.kv_off, tdev.kv_len, tplan.max_kv))
            # history token j of caption n is out[1 + j, n]
            self._ban(ws.logits, n_valid, out[1:], N, 1, t)
            if sampling is None:
                ops.rank_topk(ws.logits, n_valid, 1, vals, out[t + 1].view(N, 1))
            else:
                ops.sample_tokens(ws.logits, n_valid, out[t + 1], step=t, **sampling)
            if stop is not None:
                stop.record(out[t + 1], stop.fin, N, t)
        if stop is not None:
            stop.fill_after(out[1:], 0)
        return _copy_to_host(out[1:]).t()

    @torch.no_grad()
    def beam_search(self, batch, beam_size, length_penalty=0.0):
        """Per caption, the best of `beam_size` beams (see beam_ids), cut at the first EOS."""
        ids, _ = self.beam_ids(batch, beam_size, length_penalty)
        return [self.cut_eos(row) for row in ids.tolist()]

    @torch.no_grad()
    def beam_ids(self, batch, beam_size, length_penalty=0.0):
        """Beam search over `max_step` steps: (ids [n_captions, max_step] int32,
        score [n_captions] fp32) on the host, the chosen beam's tokens and its sum of
        log-probabilities.

        Every caption starts with beam 0 at score 0 and the other beams at -inf. At each step a
        live beam offers its top-`beam_size` tokens (descending logit, ties to the lower id) at
        score + log-probability, a finished beam (one that has emitted EOS) offers EOS at its
        score, and the caption keeps the `beam_size` best candidates (ties to the lower parent *
        beam_size + rank). The chosen beam maximises score / len ** length_penalty, len = tokens up
        to and including the first EOS (max_step without one), ties to the lower beam. With
        beam_size 1 this is greedy decoding up to the first EOS, after which it emits EOS.

        Rows n * beam_size + b run through the decoder together; the KV cache is laid out
        [max_step, rows, 3H] per layer and each beam reads its history through a KV-ancestry
        table, so nothing is copied when beams are reordered. Every upload of the batch happens
        before the loop; token histories, scores and lengths come back in one device->host copy.

        With early_stop the loop ends once every beam of every caption has finished, and the result
        is bitwise the full run's: from then on a step only re-emits EOS at unchanged scores, and
        since the beams are already in (score descending, candidate ascending) order, each new beam
        b is the old beam b, so the remaining history columns are EOS and nothing else changes. A
        beam that never finishes (one left at -inf, say) means no early stop."""
        model, T, B = self.model, int(self.max_step), int(beam_size)

        def check(n_valid):
            if not 1 <= B <= min(ops.BEAM_MAX, n_valid):
                raise ValueError(f"beam_size = {beam_size}: beam search takes 1 to "
                                 f"{min(ops.BEAM_MAX, n_valid)} beams")
            if not float(length_penalty) >= 0.0:
                raise ValueError(f"length_penalty = {length_penalty}: must be >= 0")

        tplan, tdev, w, cross, ws = self._prepare(batch, "beam search",
                                                  lambda p: p.beam_arrays(T, B), B, check)
        device, N, H = ws.x.device, tplan.n_seg, ws.x.shape[1]
        R = N * B
        n_valid = w["n_valid"]
        caches = [torch.empty(T, R, 3 * H, dtype=BF16, device=device) for _ in w["layers"]]
        rows = [c.view(T * R, 3 * H) for c in caches]
        # beam state, ping-pong over steps: [token history R x T | score | finished | length]
        slabs = [torch.empty(R * T + 3 * R, dtype=torch.int32, device=device) for _ in range(2)]
        ancs = [torch.empty(R * T, dtype=torch.int32, device=device) for _ in range(2)]
        ids = torch.full((R,), int(self.bos), dtype=torch.int32, device=device)
        lse = torch.empty(R, dtype=torch.float32, device=device)
        logp = torch.empty(R, B, dtype=torch.float32, device=device)
        cols = torch.empty(R, B, dtype=torch.int32, device=device)
        state, anc = tdev.beam_state0, tdev.beam_anc0
        stop = _EarlyStop(device, int(self.eos)) if self.early_stop else None
        for t in range(T):
            if stop is not None and t and stop.reached():
                break
            step = slice(t * R, (t + 1) * R)
            model._positions(w, ws, ids, tdev.beam_step_pos[step], R, w["layers"],
                             lambda l: (caches[l][t], rows[l][:, H:2 * H], rows[l][:, 2 * H:]),
                             model._self_attn_gather(anc.view(R, T), tdev.beam_step_len[step],
                                                     t + 1),
                             cross, (tdev.beam_kv_off, tdev.beam_kv_len, tplan.max_kv))
            # each live beam's own history: token j of row r is hist[r * T + j]
            self._ban(ws.logits, n_valid, _beam_state(state, R, T)[3], 1, T, t)
            ops.beam_logprob_topk(ws.logits, n_valid, B, lse, logp, cols)
            ops.beam_select(logp, cols, _beam_state(state, R, T), anc,
                            _beam_state(slabs[t % 2], R, T), ancs[t % 2], ids, beam=B, step=t,
                            max_step=T, eos=int(self.eos))
            state, anc = slabs[t % 2], ancs[t % 2]
            if stop is not None:
                stop.record(None, _beam_state(state, R, T)[1], R, t)
        if stop is not None:
            stop.fill_after(_beam_state(state, R, T)[3].view(R, T), 1)
        score, _, length, hist = _beam_state(_copy_to_host(state), R, T)
        best = self.pick_beam(score.view(N, B).numpy(), length.view(N, B).numpy(), length_penalty)
        sel = torch.from_numpy(np.arange(N) * B + best)
        return hist.view(R, T)[sel].clone(), score[sel].clone()

    @staticmethod
    def pick_beam(score, length, length_penalty):
        """Per caption (row), the beam maximising score / length ** length_penalty in fp64, ties
        to the lower beam."""
        norm = np.asarray(score, np.float64) / np.power(np.asarray(length, np.float64),
                                                        float(length_penalty))
        return np.argmax(norm, axis=1)

    def cut_eos(self, ids):
        out_ids = []
        for i in ids:
            if i == self.eos:
                break
            out_ids.append(i)
        return out_ids


def sampling_seed(seed, rank, index):
    """The 32-bit sampling seed of batch `index` of data-parallel rank `rank` under the user's
    `seed` (an integer in [0, 2**32)): hash_u32(hash_u32(seed, rank), index) with the dropout hash
    of csrc/ptx.cuh, so no two (rank, batch) pairs draw from the same uniforms."""
    _check_seed(seed)
    return _hash_u32(_hash_u32(int(seed), rank), index)


def _check_seed(seed):
    if int(seed) != seed or not 0 <= seed < 2 ** 32:
        raise ValueError(f"seed = {seed}: must be an integer in [0, 2**32)")


def _hash_u32(key, idx):
    m = 0xFFFFFFFF
    h = ((idx * 0x9E3779B1) & m) ^ key
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & m
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & m
    h ^= h >> 16
    return h


def _copy_to_host(x):
    """`x` on the host in one copy: into pinned memory with an event wait (no stream sync)."""
    if x.device.type != "cuda":
        return x.clone()
    host = torch.empty(x.shape, dtype=x.dtype, pin_memory=True)
    host.copy_(x, non_blocking=True)
    done = torch.cuda.Event()
    done.record()
    done.synchronize()
    return host


class _EarlyStop:
    """The stop step of one decode loop: `dev` (device int32, ops.DEC_STOP_UNSET until every row
    has ended) and its mirror `host` (pinned int32, -1 until then), which the host reads with a
    plain load. `fin` holds the per-row flags of greedy decoding and sampling (`rows` > 0)."""

    def __init__(self, device, eos, rows=0):
        self.eos = eos
        self.host = torch.empty(1, dtype=torch.int32, pin_memory=device.type == "cuda")
        self.host.fill_(-1)
        self._word = self.host.numpy()
        self.dev = torch.full((1,), ops.DEC_STOP_UNSET, dtype=torch.int32, device=device)
        self.fin = torch.zeros(rows, dtype=torch.int32, device=device) if rows else None

    def reached(self):
        return int(self._word[0]) >= 0

    def record(self, ids, fin, rows, t):
        ops.dec_finished(ids, fin, self.dev, self.host, rows=rows, eos=self.eos, step=t)

    def fill_after(self, x, step_dim):
        """EOS into every position of x whose index along `step_dim` is past the device's stop
        step (none without one), enqueued against the device scalar: no synchronisation."""
        steps = torch.arange(x.shape[step_dim], dtype=torch.int32, device=x.device)
        shape = [1] * x.dim()
        shape[step_dim] = -1
        x.masked_fill_(steps.view(shape) > self.dev, self.eos)


def _beam_state(buf, R, T):
    """(score fp32 [R], finished [R], length [R], token history [R * T]) views of one beam-state
    buffer (int32 [R * T + 3 * R], TvcPlan.beam_arrays' `beam_state0` layout)."""
    h = R * T
    return buf[h:h + R].view(torch.float32), buf[h + R:h + 2 * R], buf[h + 2 * R:], buf[:h]
