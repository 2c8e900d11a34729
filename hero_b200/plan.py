"""Host-side packing plans: padded reference batch layout -> packed (valid-token-only) layout.

The reference pads every subtitle row to the batch maximum and masks padded keys with -10000
(model/layers.py:299-302); it also re-packs `[frames | pad | text | pad]` into `[frames, text,
pad]` with torch.gather (model/encoder.py:271-279, index from data/data.py:504-512) and scatters
frame outputs back to the clip timeline in a Python double loop (model/model.py:156-187). Here all
of that becomes index arithmetic done ONCE per batch on the host with numpy; the CUDA kernels then
only ever see valid tokens:

    SeqPlan   which (row, position) pairs are valid, in row-major order -> packed token ids,
              cu_seqlens for the attention kernel, maps for pack / unpack.
    FPlan     cross-modal rows: per packed token its source (frame slot or text slot).
    CPlan     clip rows + the CSR maps replacing collect_frame_outputs (forward gather-sum and its
              transpose for the backward).

Plans are pure numpy (testable without a GPU); `.to(device)` uploads the int32 index arrays in
one pinned-memory copy.
"""
import numpy as np
import torch


ATTN_TILE = 128        # tokens per tensor-core attention tile
ATTN_TILE_SEQS = 16    # sequences per tile (one K = 16 membership step of the S MMA, csrc/attention_tc.cu)
ATTN_LONG_MAX = 768    # longest sequence the long-sequence kernels take (hero_attn_fwd)


def _np(t):
    if torch.is_tensor(t):
        return t.detach().cpu().numpy()
    return np.asarray(t)


def _max_vl_of(batch):
    """Padded number of frame slots per subtitle row: from the plan inputs, the frame features, or
    (batches without f_v_feats) the (1, max_vl) frame position ids of the collate."""
    if "_max_vl" in batch:
        return int(batch["_max_vl"])
    fv = batch.get("f_v_feats") if hasattr(batch, "get") else batch["f_v_feats"]
    if fv is not None:
        return int(fv.shape[1])
    return int(batch["f_v_pos_ids"].shape[-1])


def _rows(t):
    """Id array -> int64 [rows, L] (a 1-D array is one row)."""
    a = np.asarray(_np(t), np.int64)
    return a.reshape(1, -1) if a.ndim == 1 else a


def _host_arrays(ts):
    """Tensors, arrays or None -> numpy arrays or None. Tensors that live on a device come back
    in ONE device->host copy."""
    on_dev = [t for t in ts if torch.is_tensor(t) and t.device.type != "cpu"]
    if not on_dev:
        return [None if t is None else _np(t) for t in ts]
    flat = torch.cat([t.reshape(-1).to(torch.int64) for t in on_dev]).cpu().numpy()
    out, o = [], 0
    for t in ts:
        if torch.is_tensor(t) and t.device.type != "cpu":
            out.append(flat[o:o + t.numel()].reshape(tuple(t.shape)))
            o += t.numel()
        else:
            out.append(None if t is None else _np(t))
    return out


class DeviceIndex:
    """A bundle of int32 index arrays uploaded to the device with a single H2D copy.

    `staging(n)` (optional) returns a reusable (pinned host, device) pair of int32 buffers with at
    least n elements. Without it every upload allocates pinned memory; under load the caching host
    allocator cannot recycle blocks whose copies are still in flight and falls back to
    cudaHostAlloc — tens of milliseconds and a device synchronisation per call (measured: 30-50 ms
    holes in the step timeline). loader.BatchStager passes its per-slot buffers."""

    def __init__(self, arrays, device, staging=None):
        names = list(arrays)
        sizes = [int(arrays[n].size) for n in names]
        offs = np.concatenate([[0], np.cumsum([(s + 3) // 4 * 4 for s in sizes])]).astype(np.int64)
        total = int(offs[-1])
        if staging is not None:
            host_buf, dev_buf = staging(total)
            host, dst = host_buf[:total], dev_buf[:total]
        else:
            host = torch.empty(total, dtype=torch.int32,
                               pin_memory=torch.cuda.is_available() and device.type == "cuda")
            dst = None
        hv = host.numpy()
        for n, o, s in zip(names, offs[:-1], sizes):
            hv[o:o + s] = arrays[n].reshape(-1)
        if dst is None:
            self.flat = host.to(device, non_blocking=True)
        else:
            dst.copy_(host, non_blocking=True)
            self.flat = dst
        self._host = host  # keep pinned memory alive until the copy is consumed
        for n, o, s in zip(names, offs[:-1], sizes):
            setattr(self, n, self.flat[o:o + s])


class SeqPlan:
    """Valid positions of a padded (rows, length) mask, packed row-major."""

    def __init__(self, mask):
        mask = _np(mask) != 0
        self.rows, self.length = mask.shape
        r, c = np.nonzero(mask)                      # row-major order
        self.tok_row = r.astype(np.int32)
        self.tok_col = c.astype(np.int32)
        self.n_tok = int(r.size)
        lens = mask.sum(1).astype(np.int64)
        self.lens = lens
        self.cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        self.n_seq = self.rows
        self.max_len = int(lens.max()) if lens.size else 0
        self.tok_flat = (r.astype(np.int64) * self.length + c).astype(np.int32)  # packed -> padded
        p2t = np.full(self.rows * self.length, -1, np.int32)
        p2t[self.tok_flat] = np.arange(self.n_tok, dtype=np.int32)
        self.pad_to_tok = p2t                                                    # padded -> packed
        # attention tiling: consecutive sequences packed into tiles of <= 128 tokens and <= 16
        # sequences (a sequence never straddles tiles); per token the [lo, hi) range of its own
        # sequence. Sequences
        # longer than one tile (up to ATTN_LONG_MAX tokens; the reference's position table allows
        # 514, model/encoder.py:50) become tiles of their own at the END of the list: the library
        # runs those `n_long` tiles on its long-sequence kernels (hero_attn_fwd).
        if self.max_len > ATTN_LONG_MAX:
            row = int(np.argmax(lens))
            raise ValueError(f"row {row} has {self.max_len} valid tokens; the attention kernels "
                             f"support sequences of up to {ATTN_LONG_MAX} tokens")
        self.seq_lo = np.repeat(self.cu[:-1], lens).astype(np.int32)
        self.seq_hi = np.repeat(self.cu[1:], lens).astype(np.int32)
        t0, tn, l0, ln = [], [], [], []
        start, cur, nseq = 0, 0, 0
        pos = 0
        for n in lens.tolist():
            if n == 0:
                continue
            if n > ATTN_TILE:
                if cur:
                    t0.append(start)
                    tn.append(cur)
                l0.append(pos)
                ln.append(n)
                pos += n
                start, cur, nseq = pos, 0, 0
                continue
            if cur + n > ATTN_TILE or nseq == ATTN_TILE_SEQS:
                t0.append(start)
                tn.append(cur)
                start, cur, nseq = start + cur, 0, 0
            cur += n
            nseq += 1
            pos += n
        if cur:
            t0.append(start)
            tn.append(cur)
        self.n_long = len(l0)
        self.max_long = max(ln) if ln else 0
        self.short_tok0, self.short_ntok = np.asarray(t0, np.int32), np.asarray(tn, np.int32)
        self.long_tok0, self.long_ntok = np.asarray(l0, np.int32), np.asarray(ln, np.int32)
        self.tile_tok0 = np.concatenate([self.short_tok0, self.long_tok0]).astype(np.int32)
        self.tile_ntok = np.concatenate([self.short_ntok, self.long_ntok]).astype(np.int32)
        self.n_tiles = len(t0) + len(l0)

    def arrays(self, prefix):
        return {prefix + "cu": self.cu, prefix + "tok_flat": self.tok_flat,
                prefix + "pad_to_tok": self.pad_to_tok, prefix + "seq_lo": self.seq_lo,
                prefix + "seq_hi": self.seq_hi, prefix + "tile_tok0": self.tile_tok0,
                prefix + "tile_ntok": self.tile_ntok}

    def attn(self, dev, prefix):
        """Device-side attention plan consumed by ops.attn_fwd / attn_bwd."""
        return {"cu": getattr(dev, prefix + "cu"), "seq_lo": getattr(dev, prefix + "seq_lo"),
                "seq_hi": getattr(dev, prefix + "seq_hi"),
                "tile_tok0": getattr(dev, prefix + "tile_tok0"),
                "tile_ntok": getattr(dev, prefix + "tile_ntok"), "n_tiles": self.n_tiles,
                "n_long": self.n_long, "max_long": self.max_long,
                "n_tok": self.n_tok, "n_seq": self.n_seq, "max_len": self.max_len}


def _csr(dst, src, n_dst):
    """CSR (offsets, indices) listing for each dst all its src, stable in src order."""
    dst = np.asarray(dst, np.int64)
    src = np.asarray(src, np.int32)
    order = np.argsort(dst, kind="stable")
    counts = np.bincount(dst, minlength=n_dst)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    return off, src[order]


class FPlan:
    """Cross-modal ('repr') rows: frames + subtitle tokens per row, or text-only rows ('txt')."""

    def __init__(self, attn_mask, gather_index=None, max_vl=0, max_sl=None):
        self.seq = SeqPlan(attn_mask)
        s = self.seq
        if gather_index is None:       # text only: position j reads text slot j
            src = s.tok_col.astype(np.int64)
            max_vl = 0
            self.max_sl = s.length if max_sl is None else max_sl
        else:
            gi = _np(gather_index).astype(np.int64)
            src = gi[s.tok_row, s.tok_col]
            self.max_sl = int(max_sl or 0)
        self.max_vl = int(max_vl)
        is_img = src < self.max_vl
        tok = np.arange(s.n_tok, dtype=np.int32)
        self.img_tok = tok[is_img]
        self.img_k = src[is_img].astype(np.int32)                       # frame slot in the row
        self.img_src = (s.tok_row[is_img].astype(np.int64) * self.max_vl
                        + src[is_img]).astype(np.int32)                 # row in f_v_feats.view(-1, D)
        self.txt_tok = tok[~is_img]
        self.txt_j = (src[~is_img] - self.max_vl).astype(np.int32)
        self.txt_src = (s.tok_row[~is_img].astype(np.int64) * self.max_sl
                        + self.txt_j).astype(np.int32)                  # index in input_ids.view(-1)
        self.n_img = int(self.img_tok.size)
        self.n_txt = int(self.txt_tok.size)
        self.n_tok = s.n_tok

    def arrays(self, prefix="f_"):
        """The attention plan under `prefix`, and the embedding arrays (`embed_ids`) unprefixed."""
        a = self.seq.arrays(prefix)
        a.update(getattr(self, "emb", {}))
        return a

    def embed_ids(self, input_ids=None, pos_ids=None, img_pos_ids=None, padding_idx=1):
        """The index arrays of functional.cross_modal_embed (`self.emb`), gathered here on the
        host: per packed text token its row (txt_tok), vocabulary id and position id; per packed
        frame token its row, feature row (img_src) and position id; and for each position table a
        CSR over the position ids the tokens read (deterministic table gradients). Missing
        `pos_ids` follow SubEmbeddings.create_position_ids_from_input_ids; missing `img_pos_ids`
        are the frame slots."""
        txt_ids = txt_pos = np.zeros(0, np.int64)
        if self.n_txt:
            ids = _rows(input_ids)
            if pos_ids is None:
                keep = ids != padding_idx
                pos = np.cumsum(keep, 1) * keep + padding_idx
            else:
                pos = _rows(pos_ids)
            txt_ids = ids.reshape(-1)[self.txt_src]
            txt_pos = pos[0][self.txt_j] if pos.shape[0] == 1 else pos.reshape(-1)[self.txt_src]
        img_pos = self.img_k if img_pos_ids is None else \
            _rows(img_pos_ids).reshape(-1)[self.img_k]
        self.emb = {"txt_tok": self.txt_tok, "txt_ids": txt_ids.astype(np.int32),
                    "img_tok": self.img_tok, "img_src": self.img_src}
        self.emb.update(pos_csr("txt", txt_pos))
        self.emb.update(pos_csr("img", img_pos))


class CPlan:
    """Clip-level rows and the frame-merge maps (collect_frame_outputs as CSR gathers)."""

    def __init__(self, c_attn_mask, fplan, num_subs, sub_idx2frame_idx):
        self.seq = SeqPlan(c_attn_mask)
        s = self.seq
        B, T = s.rows, s.length
        self.c_src = s.tok_flat                       # row in c_v_feats.view(-1, D)
        self.c_t = s.tok_col                          # temporal position id
        # (clip, frame) <- (sub row, slot k): model/model.py:171-186
        rows, ks, dst = [], [], []
        start = 0
        for vid, n_sub in enumerate(num_subs):
            for sid, frames in sub_idx2frame_idx[vid]:
                n = len(frames)
                if n:
                    rows.extend([start + sid] * n)
                    ks.extend(range(n))
                    dst.extend(vid * T + int(t) for t in frames)
            start += n_sub
        rows = np.asarray(rows, np.int64)
        ks = np.asarray(ks, np.int64)
        dst = np.asarray(dst, np.int64)
        if dst.size and (dst.max() >= B * T or dst.min() < 0):
            raise IndexError("sub_idx2frame_idx refers to a frame outside the clip tensor")
        # (sub row, slot) -> row of c_v_feats.view(-1, D); -1 where the slot holds no clip frame
        self.frame_source = np.full(fplan.seq.rows * max(fplan.max_vl, 1), -1, np.int32)
        if rows.size:
            self.frame_source[rows * fplan.max_vl + ks] = dst
        f_tok = fplan.seq.pad_to_tok[rows * fplan.seq.length + ks] if rows.size else \
            np.zeros(0, np.int32)
        c_tok = s.pad_to_tok[dst] if dst.size else np.zeros(0, np.int32)
        keep = (f_tok >= 0) & (c_tok >= 0)            # masked slots carry no defined value
        f_tok, c_tok = f_tok[keep], c_tok[keep]
        self.n_pairs = int(f_tok.size)
        self.fwd_off, self.fwd_idx = _csr(c_tok, f_tok, s.n_tok)             # c token <- f tokens
        self.bwd_off, self.bwd_idx = _csr(f_tok, c_tok, fplan.seq.n_tok)     # f token <- c tokens

    def arrays(self, prefix="c_"):
        a = self.seq.arrays(prefix)
        a.update({prefix + "src": self.c_src, prefix + "t": self.c_t,
                  prefix + "fwd_off": self.fwd_off, prefix + "fwd_idx": self.fwd_idx,
                  prefix + "bwd_off": self.bwd_off, prefix + "bwd_idx": self.bwd_idx})
        return a


def table_csr(idx, n_rows):
    """CSR listing, for every embedding-table row, the packed tokens that used it (deterministic
    table gradients via gather-sum instead of contended atomics)."""
    idx = np.asarray(idx, np.int64)
    return _csr(idx, np.arange(idx.size, dtype=np.int32), n_rows)


def pos_csr(name, pos):
    """`{name}_pos` (per-token position ids, int32) and the `table_csr` over them,
    `{name}pos_off / idx`, covering the table rows up to the largest id used."""
    pos = np.asarray(pos, np.int32)
    off, idx = table_csr(pos, int(pos.max()) + 1 if pos.size else 1)
    return {name + "_pos": pos, name + "pos_off": off, name + "pos_idx": idx}


class ReprPlan:
    """Everything HierarchicalVlModel.forward_repr needs for one batch (a `plan_inputs` dict)."""

    def __init__(self, batch):
        # `plan_inputs` dicts carry the two padded lengths instead of the big tensors
        max_vl = _max_vl_of(batch)
        max_sl = batch["_max_sl"] if "_max_sl" in batch else batch["f_sub_input_ids"].shape[1]
        self.f = FPlan(batch["f_attn_masks"], batch["f_gather_index"], max_vl, max_sl)
        self.c = CPlan(batch["c_attn_masks"], self.f, batch["num_subs"],
                       batch["sub_idx2frame_idx"])
        # Every frame slot of a subtitle row is a copy of a clip frame (data/data.py:380-395 fills
        # f_v_feats with index_select(c_v_feats, frames)): row of c_v_feats.view(-1, D) behind each
        # packed frame token, so a batch may omit `f_v_feats` altogether (half the H2D bytes).
        self.f.img_src_c = self.c.frame_source[self.f.img_src] if self.f.n_img else \
            np.zeros(0, np.int32)
        # a frame slot that is valid in f_attn_masks but not listed in sub_idx2frame_idx has no
        # clip frame behind it: such a batch must ship its own f_v_feats (checked on the host, the
        # LayerNorm kernels index x_rows without a sign test)
        self.f.shared_feats_ok = self.shared_feats_ok = bool((self.f.img_src_c >= 0).all())
        self.shape_f = tuple(batch["f_attn_masks"].shape)
        self.shape_c = tuple(batch["c_attn_masks"].shape)
        # position-table CSR of the temporal embeddings
        self.c_pos_off, self.c_pos_idx = table_csr(self.c.c_t, max(self.shape_c[1], 1))
        get = batch.get if hasattr(batch, "get") else (lambda k: None)
        self.f.embed_ids(get("f_sub_input_ids"), get("f_sub_pos_ids"), get("f_v_pos_ids"))
        self.f.emb["img_src_c"] = self.f.img_src_c
        self.dev = None

    def to(self, device, staging=None):
        if self.dev is None or self.dev.flat.device != torch.device(device):
            a = self.f.arrays("f_")
            a.update(self.c.arrays("c_"))
            a.update({"c_pos_off": self.c_pos_off, "c_pos_idx": self.c_pos_idx})
            self.dev = DeviceIndex(a, torch.device(device), staging)
        return self.dev


class TxtPlan:
    """Rows of a CrossModalTrm pass without the clip level: text-only rows (the 'txt' task; with
    no `input_ids`, the generic BertEncoder API, which needs no embedding arrays) or, with
    `gather_index`, the frame + text rows of an MLM batch (data/mlm.py mlm_collate). Built from
    `plan_inputs(batch, "txt")` or `plan_inputs(batch, "mlm")`."""

    def __init__(self, attn_mask, input_ids=None, pos_ids=None, gather_index=None,
                 img_pos_ids=None, max_vl=0):
        max_sl = None if input_ids is None else input_ids.shape[1]
        self.f = FPlan(attn_mask, gather_index, max_vl, max_sl)
        self.shape = tuple(_np(attn_mask).shape)
        if input_ids is not None or self.f.n_txt == 0:
            self.f.embed_ids(input_ids, pos_ids, img_pos_ids)
        self.dev = None

    def to(self, device, staging=None):
        if self.dev is None or self.dev.flat.device != torch.device(device):
            self.dev = DeviceIndex(self.f.arrays("f_"), torch.device(device), staging)
        return self.dev


class JointPlan:
    """Video rows ('repr') and text-only query rows ('txt') of the SAME CrossModalTrm concatenated
    into one packed token stream, so both go through the 6 layers as one set of GEMMs (32 query
    rows x 16 tokens alone would run every GEMM at M = 512, ~10 % tensor utilisation).
    Query tokens follow the video tokens: packed index = n_video_tokens + query index."""

    def __init__(self, rplan, tplan):
        self.r, self.t = rplan, tplan
        fv, fq = rplan.f, tplan.f
        a = fv.seq.n_tok
        self.n_video_tok = a
        self.n_tok = a + fq.seq.n_tok
        self.n_txt = fv.n_txt + fq.n_txt
        self.n_img = fv.n_img
        self.shared_feats_ok = rplan.shared_feats_ok
        sv, sq = fv.seq, fq.seq
        self.n_seq = sv.n_seq + sq.n_seq
        self.max_len = max(sv.max_len, sq.max_len)
        self.n_tiles = sv.n_tiles + sq.n_tiles
        # long-sequence tiles (rare) of both row kinds go last, after every 128-token tile
        self.n_long = sv.n_long + sq.n_long
        self.max_long = max(sv.max_long, sq.max_long)
        if not hasattr(fq, "emb"):
            raise ValueError("the query plan was built without input_ids: build it with "
                             "TxtPlan(**plan_inputs(batch, 'txt'))")
        ev, eq = fv.emb, fq.emb
        self.arr = {
            "j_cu": np.concatenate([sv.cu, sq.cu[1:] + a]).astype(np.int32),
            "j_seq_lo": np.concatenate([sv.seq_lo, sq.seq_lo + a]).astype(np.int32),
            "j_seq_hi": np.concatenate([sv.seq_hi, sq.seq_hi + a]).astype(np.int32),
            "j_tile_tok0": np.concatenate([sv.short_tok0, sq.short_tok0 + a, sv.long_tok0,
                                           sq.long_tok0 + a]).astype(np.int32),
            "j_tile_ntok": np.concatenate([sv.short_ntok, sq.short_ntok, sv.long_ntok,
                                           sq.long_ntok]).astype(np.int32),
            "txt_tok": np.concatenate([ev["txt_tok"], eq["txt_tok"] + a]).astype(np.int32),
            "txt_ids": np.concatenate([ev["txt_ids"], eq["txt_ids"]]).astype(np.int32),
        }
        self.arr.update(pos_csr("txt", np.concatenate([ev["txt_pos"], eq["txt_pos"]])))
        self.arr.update({k: v for k, v in ev.items() if k.startswith("img")})
        self.dev = None

    def to(self, device, staging=None):
        device = torch.device(device)
        if self.dev is None or self.dev.flat.device != device:
            self.dev = DeviceIndex(self.arr, device, staging)
        return self.dev

    def attn(self, dev):
        return {"cu": dev.j_cu, "seq_lo": dev.j_seq_lo, "seq_hi": dev.j_seq_hi,
                "tile_tok0": dev.j_tile_tok0, "tile_ntok": dev.j_tile_ntok,
                "n_tiles": self.n_tiles, "n_long": self.n_long, "max_long": self.max_long,
                "n_tok": self.n_tok, "n_seq": self.n_seq, "max_len": self.max_len}


class QaPlan:
    """Query-fused temporal rows of video QA (model/videoQA.py:68-86): row r = (video v, candidate
    q) of the collate (video-major, Nq = rows / Nv) is [valid frames of c_attn_masks[r] | valid
    tokens of qa_attn_masks[r]], each sequence contiguous in one packed buffer. Frames keep their
    column as temporal position; question / answer tokens take `qa_pos_ids`.

    Frame tokens appear in the same row-major order as CPlan's clip tokens, so frame k of the
    packed stream reads row k of the cross-modal output `g` (no source map needed).

    VIOLIN (model/violin.py:50-70) has the same rows with a statement in place of question +
    answer: built with n_videos = rows, so Nq = 1 and each statement row pools its own frames."""

    def __init__(self, c_attn_masks, qa_attn_masks, qa_input_ids, qa_pos_ids, n_videos):
        cm, qm = _np(c_attn_masks) != 0, _np(qa_attn_masks) != 0
        rows, L = cm.shape
        if qm.shape[0] != rows:
            raise ValueError(f"qa_attn_masks has {qm.shape[0]} rows, c_attn_masks {rows}")
        if n_videos < 1 or rows % n_videos:
            raise ValueError(f"{rows} query-fused rows do not split into {n_videos} videos")
        self.n_videos, self.n_cand, self.length = int(n_videos), rows // int(n_videos), L
        # attention tiles of the joint rows; a row over ATTN_LONG_MAX tokens raises here
        self.seq = SeqPlan(np.concatenate([cm, qm], 1))
        s = self.seq
        tok = np.arange(s.n_tok, dtype=np.int32)
        is_frm = s.tok_col < L
        self.frm_tok = tok[is_frm]                                    # packed row of frame k
        self.frm_t = s.tok_col[is_frm].astype(np.int32)               # its temporal position
        self.qa_tok = tok[~is_frm]
        qa_row, qa_j = s.tok_row[~is_frm], (s.tok_col[~is_frm] - L).astype(np.int64)
        ids = np.asarray(_np(qa_input_ids), np.int64)
        pos = np.asarray(_np(qa_pos_ids), np.int64)
        pos = pos.reshape(1, -1) if pos.ndim == 1 else pos
        self.qa_ids = ids[qa_row, qa_j].astype(np.int32)
        self.qa_pos = (pos[0][qa_j] if pos.shape[0] == 1 else pos[qa_row, qa_j]).astype(np.int32)
        self.n_frm, self.n_qa = int(self.frm_tok.size), int(self.qa_tok.size)
        # deterministic position-table gradients: CSR over the position ids actually used
        self.cpos_off, self.cpos_idx = table_csr(self.frm_t, max(L, 1))
        n_qpos = int(self.qa_pos.max()) + 1 if self.n_qa else 1
        self.qpos_off, self.qpos_idx = table_csr(self.qa_pos, n_qpos)
        # (v, q, l) -> packed row of that frame, -1 for padding (read by the pooling kernels)
        fmap = np.full(rows * L, -1, np.int32)
        fmap[s.tok_row[is_frm].astype(np.int64) * L + self.frm_t] = self.frm_tok
        self.frame_map = fmap
        self.n_long_rows = int(s.n_long)
        self.dev = None

    def to(self, device, staging=None):
        device = torch.device(device)
        if self.dev is None or self.dev.flat.device != device:
            a = {"cu": self.seq.cu, "seq_lo": self.seq.seq_lo, "seq_hi": self.seq.seq_hi,
                 "tile_tok0": self.seq.tile_tok0, "tile_ntok": self.seq.tile_ntok,
                 "frm_tok": self.frm_tok, "frm_t": self.frm_t, "qa_tok": self.qa_tok,
                 "qa_ids": self.qa_ids, "qa_pos": self.qa_pos, "cpos_off": self.cpos_off,
                 "cpos_idx": self.cpos_idx, "qpos_off": self.qpos_off, "qpos_idx": self.qpos_idx,
                 "frame_map": self.frame_map}
            self.dev = DeviceIndex(a, device, staging)
        return self.dev

    def attn(self, dev):
        return self.seq.attn(dev, "")


PLAN_KEY = "_hero_plan"
QA_PLAN_KEY = "_hero_qa_plan"
QUERY_PLAN_KEY = "_hero_query_plan"
_REPR_KEYS = ("f_attn_masks", "f_gather_index", "c_attn_masks", "f_sub_input_ids",
              "f_sub_pos_ids", "f_v_pos_ids")
# TxtPlan arguments and the batch keys they come from, per kind
_TXT_ARGS = ("attn_mask", "input_ids", "pos_ids", "gather_index", "img_pos_ids")
_TXT_KEYS = {"txt": ("attn_masks", "input_ids", "pos_ids", None, None),
             "mlm": ("attn_masks", "input_ids", "position_ids", "gather_index", "f_pos_ids")}
# key prefix of the query-fused text of each kind: question + answer rows of video QA, the
# statement rows of VIOLIN
_QA_PREFIX = {"videoqa": "qa", "violin": "q"}
_QA_ARGS = ("qa_attn_masks", "qa_input_ids", "qa_pos_ids")


def _qa_keys(prefix):
    return tuple(prefix + k[2:] for k in _QA_ARGS)


def plan_inputs(batch, kind="repr"):
    """The small, picklable part of a batch that a plan is built from: masks and id tensors as
    host arrays, index lists and padded lengths; none of the feature tensors. Every plan is built
    from it, in collate workers, PlanPool processes or, without an attached plan, in the forward;
    tensors that live on the device come back in ONE device->host copy.
    kind: 'repr' (video batch), 'videoqa' / 'violin' (+ the QaPlan arguments under "_qa"),
    'txt' (query batch) or 'mlm' (data/mlm.py batch): the last two give TxtPlan's arguments."""
    get = batch.get if hasattr(batch, "get") else batch.__getitem__
    if kind in _TXT_KEYS:
        keys = _TXT_KEYS[kind]
        d = dict(zip(_TXT_ARGS, _host_arrays([None if k is None else get(k) for k in keys])))
        if d["gather_index"] is not None:
            d["max_vl"] = int(batch["v_feat"].shape[1])
        return d
    keys = _REPR_KEYS + (_qa_keys(_QA_PREFIX[kind]) if kind in _QA_PREFIX else ())
    d = dict(zip(keys, _host_arrays([get(k) for k in keys])))
    for k in ("num_subs", "sub_idx2frame_idx"):
        d[k] = _np(batch[k]) if torch.is_tensor(batch[k]) else batch[k]
    d["_max_vl"] = _max_vl_of(batch)
    d["_max_sl"] = int(batch["f_sub_input_ids"].shape[1])
    if kind in _QA_PREFIX:
        qa = [d.pop(k) for k in keys[len(_REPR_KEYS):]]
        d["_qa"] = dict(zip(_QA_ARGS, qa), c_attn_masks=d["c_attn_masks"],
                        n_videos=int(batch["targets"].shape[0]))
    return d


def build_plans(repr_in, txt_in=None):
    """ReprPlan (+ TxtPlan and the JointPlan of the fused video+query pass) from `plan_inputs`
    dicts. Pure numpy: runs in collate workers / PlanPool processes. A video QA or VIOLIN batch's
    QaPlan rides along as `rplan._qa` (PlanPool.attach stores it under QA_PLAN_KEY)."""
    rplan = ReprPlan(repr_in)
    if repr_in.get("_qa") is not None:
        rplan.__dict__["_qa"] = QaPlan(**repr_in["_qa"])
    if txt_in is None:
        return rplan, None
    tplan = TxtPlan(**txt_in)
    rplan.__dict__["_joint"] = JointPlan(rplan, tplan)
    return rplan, tplan


class PlanPool:
    """Builds plans in worker processes, the way the reference builds its gather indices inside
    DataLoader collate workers (data/data.py video_collate, model/model.py:189-193) — the training
    process only uploads the finished index arrays. `submit` returns a future whose `result()` is
    (ReprPlan, TxtPlan | None); `attach(future, batch, txt_batch)` stores them in the batch dicts."""

    def __init__(self, workers=2):
        import concurrent.futures as cf
        import multiprocessing as mp
        self._ex = cf.ProcessPoolExecutor(max_workers=workers, mp_context=mp.get_context("spawn"))

    def submit(self, batch, txt_batch=None):
        return self._ex.submit(build_plans, plan_inputs(batch, video_kind(batch)),
                               None if txt_batch is None else plan_inputs(txt_batch, "txt"))

    @staticmethod
    def attach(future, batch, txt_batch=None):
        rplan, tplan = future.result()
        batch[PLAN_KEY] = rplan
        qplan = rplan.__dict__.pop("_qa", None)
        if qplan is not None:
            batch[QA_PLAN_KEY] = qplan
        if txt_batch is not None:
            txt_batch[PLAN_KEY] = tplan
        return batch, txt_batch

    def shutdown(self):
        self._ex.shutdown(wait=False, cancel_futures=True)


def attach_plan(batch, kind="repr"):
    """Collate-side hook: build the plan from HOST tensors (no device sync later) and stash it in
    the batch dict; `move_to_cuda`-style helpers leave non-tensor values alone.
    kind: 'repr' (video batch), 'txt' (query batch), 'mlm' (data/mlm.py batch), 'vsm' — a VSM /
    VCMR training batch that carries its queries as `query_input_ids / query_pos_ids /
    query_attn_masks` (data/vcmr.py): attaches the video plan, the query plan (QUERY_PLAN_KEY) and
    their joint plan — or 'videoqa' (data/videoQA.py video_qa_collate) / 'violin'
    (data/violin.py violin_collate): the video plan of the cross-modal rows and the QaPlan of the
    query-fused temporal rows (QA_PLAN_KEY).
    The plan captures the batch's token / position ids per packed token (FPlan.embed_ids): attach
    it AFTER any masking of `input_ids` (the reference masks in the dataset, before collate), and
    attach again if the ids are edited afterwards."""
    if kind in _TXT_KEYS:
        batch[PLAN_KEY] = TxtPlan(**plan_inputs(batch, kind))
        return batch
    query = None
    if kind == "vsm":
        query = plan_inputs({k: batch.get("query_" + k) for k in _TXT_KEYS["txt"][:3]}, "txt")
    rplan, tplan = build_plans(plan_inputs(batch, "repr" if kind == "vsm" else kind), query)
    batch[PLAN_KEY] = rplan
    if tplan is not None:
        batch[QUERY_PLAN_KEY] = tplan
    if "_qa" in rplan.__dict__:
        batch[QA_PLAN_KEY] = rplan.__dict__.pop("_qa")
    return batch


def video_kind(batch):
    """'videoqa' for a video_qa_collate batch (it carries question / answer rows), 'violin' for a
    violin_collate batch (statement rows), else 'repr'."""
    get = batch.get if hasattr(batch, "get") else (lambda k: None)
    for kind, prefix in _QA_PREFIX.items():
        if get(f"{prefix}_attn_masks") is not None:
            return kind
    return "repr"


def qa_plan(batch, prefix="qa"):
    """QaPlan of a video_qa_collate batch (prefix "qa") or a violin_collate batch ("q")."""
    keys = ("c_attn_masks",) + _qa_keys(prefix)
    return QaPlan(*_host_arrays([batch[k] for k in keys]), int(batch["targets"].shape[0]))


class TvcPlan:
    """Caption segments of a TVC batch (model/tvc.py:219-238, data/tvc.py:100-161): segment s of
    the flattened `clip_ranges` is the frames [st, ed) of its video. Instead of padding the segments
    to (n_seg, Lv, H), the plan lists the packed clip-level rows of every segment's frames
    (CSR `seg_off` into `seg_src`); the decoder's cross-attention K / V are computed once per layer
    over those gathered rows, and caption s attends to rows [kv_off[s], kv_off[s] + kv_len[s]).

    An empty segment (st == ed == nframes when the caption starts past the last frame,
    data/tvc.py:119-138) is all padding in the reference, masked uniformly, so its cross-attention
    returns exactly the value bias. `seg_src` ends with one extra -1 entry, a zero input row whose
    K / V are the biases; empty segments attend to it alone. A batch whose segments are all empty
    raises ValueError. Built on the host from `clip_ranges` (a host tuple) and the ReprPlan: no
    device read-back."""

    def __init__(self, clip_ranges, rplan):
        s = rplan.c.seq
        segs = [(v, int(st), int(ed)) for v, rs in enumerate(clip_ranges) for st, ed in rs]
        if len(clip_ranges) != s.rows:
            raise ValueError(f"clip_ranges lists {len(clip_ranges)} videos, the batch has {s.rows}")
        if not segs:
            raise ValueError("the batch has no caption segment")
        src, off, lens = [], [], []
        n = 0
        for v, st, ed in segs:
            if not 0 <= st <= ed <= int(s.lens[v]):
                raise ValueError(f"segment [{st}, {ed}) of video {v} is outside its "
                                 f"{int(s.lens[v])} frames")
            rows = s.pad_to_tok[v * s.length + np.arange(st, ed)]
            if (rows < 0).any():
                raise ValueError(f"segment [{st}, {ed}) of video {v} covers a masked frame")
            src.append(rows)
            off.append(n)
            lens.append(ed - st)
            n += ed - st
        if n == 0:
            raise ValueError("every caption segment of the batch is empty; the decoder needs at "
                             "least one frame to attend to")
        self.n_seg = len(segs)
        self.n_rows = n + 1                                   # + the zero row of empty segments
        self.seg_src = np.concatenate(src + [np.array([-1])]).astype(np.int32)
        self.seg_off = np.concatenate([off, [n]]).astype(np.int32)
        lens = np.asarray(lens, np.int32)
        self.seg_len = lens
        self.kv_off = np.where(lens > 0, self.seg_off[:-1], n).astype(np.int32)
        self.kv_len = np.maximum(lens, 1).astype(np.int32)
        self.max_kv = int(self.kv_len.max())
        self.dev = None

    def decode_arrays(self, max_step):
        """Per-step index arrays of greedy decoding over a KV cache laid out [n_seg, max_step, *]:
        `self_off` [n_seg] (first cache row of each caption), `step_len` [max_step, n_seg] (keys
        0..t at step t), `step_pos` [max_step, n_seg] (position id t)."""
        n, t = self.n_seg, np.arange(max_step, dtype=np.int32)
        return {"self_off": (np.arange(n, dtype=np.int32) * max_step).astype(np.int32),
                "step_len": np.repeat(t + 1, n).astype(np.int32),
                "step_pos": np.repeat(t, n).astype(np.int32)}

    def beam_arrays(self, max_step, beam):
        """Index arrays of beam search over R = n_seg * beam rows (row n * beam + b is beam b of
        caption n) with a KV cache laid out [max_step, R, *]: each caption's cross-attention range
        repeated per beam (`beam_kv_off` / `beam_kv_len` [R]), per-step position ids and
        self-attention lengths (`beam_step_pos` / `beam_step_len` [max_step, R]: t and t + 1), the
        initial state `beam_state0` in the layout of one beam-state buffer (token history [R,
        max_step] zeros, then the scores' fp32 bits (0 for beam 0, -inf for the others), finished
        flags and lengths [R] each, zeros), and the initial KV-ancestry table `beam_anc0` [R,
        max_step] whose column 0 is the row each beam writes at step 0, r."""
        R, T = self.n_seg * beam, max_step
        t = np.arange(T, dtype=np.int32)
        score = np.where(np.arange(R) % beam == 0, 0.0, -np.inf).astype(np.float32)
        anc = np.zeros((R, T), np.int32)
        anc[:, 0] = np.arange(R, dtype=np.int32)
        return {"beam_kv_off": np.repeat(self.kv_off, beam).astype(np.int32),
                "beam_kv_len": np.repeat(self.kv_len, beam).astype(np.int32),
                "beam_step_pos": np.repeat(t, R).astype(np.int32),
                "beam_step_len": np.repeat(t + 1, R).astype(np.int32),
                "beam_state0": np.concatenate([np.zeros(R * T, np.int32), score.view(np.int32),
                                               np.zeros(2 * R, np.int32)]),
                "beam_anc0": anc.reshape(-1)}

    def forced_arrays(self, length):
        """Index arrays of a teacher-forced pass over (n_seg, length) caption rows, row-major:
        causal self-attention ranges and each row's cross-attention range."""
        n = self.n_seg
        t = np.tile(np.arange(length, dtype=np.int32), n)
        return {"tf_self_off": np.repeat(np.arange(n, dtype=np.int64) * length, length)
                .astype(np.int32),
                "tf_self_len": (t + 1).astype(np.int32),
                "tf_kv_off": np.repeat(self.kv_off, length).astype(np.int32),
                "tf_kv_len": np.repeat(self.kv_len, length).astype(np.int32)}

    def to(self, device, extra=None, staging=None):
        """Upload the segment maps and `extra` (decode_arrays / forced_arrays) in one copy."""
        a = {"seg_src": self.seg_src, "kv_off": self.kv_off, "kv_len": self.kv_len}
        a.update(extra or {})
        return DeviceIndex(a, torch.device(device), staging)
