"""TEST INFRASTRUCTURE: torch restatements of the TVC decoding-control entry points
(include/hero_b200.h: hero_dec_ban_tokens, hero_sample_tokens), in the style of
tests/fake_beam_ops.py, so the controls and sampling run on a CPU-only box. Also used on the GPU as
the restatements the kernels are checked against.

The rules, as csrc/decode_ctl.cu states them:
  bans at step t of row r, s = [bos, y_0 .. y_{t-1}], L = t + 1: with n >= 1 and L >= n, token
  s[j + n - 1] is banned for every j in [0, L - n] with s[j .. j + n - 2] == s[L - n + 1 .. L - 1];
  with t < min_length, eos is banned. Banned columns c < n_valid get -inf.
  sampling of row r at step t: x = z / temperature (fp32); top-k keeps key(x) >= the k-th largest
  key (0 < k < n); top-p keeps key(x) >= theta, the largest key whose kept columns at or above it
  weigh >= max(1, ceil(p * W)) with w = floor(exp(x - max x) * 2^32) and W their sum; the id is the
  argmax over the kept columns with x_j > -inf of x_j + G_j, ties to the lower j, with
    rkey = hash_u32(hash_u32(seed, r), t)
    u_j  = ((hash_u32(rkey, j) >> 9) + 0.5) * 2^-23,   G_j = -log(-log(u_j))
  (every u_j lies strictly inside (0, 1), so G_j is finite).
"""
import math

import torch

M32 = 0xFFFFFFFF


def hash_u32(key, idx):
    """csrc/ptx.cuh hash_u32 on int64 tensors (or ints) holding uint32 values."""
    h = ((idx * 0x9E3779B1) & M32) ^ key
    h = h ^ (h >> 16)
    h = (h * 0x85EBCA6B) & M32
    h = h ^ (h >> 13)
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def ord_key(x):
    """Order-preserving uint32 image of fp32 values, as int64."""
    b = x.float().contiguous().view(torch.int32).long() & M32
    return torch.where(b >= 0x80000000, (~b) & M32, b | 0x80000000)


def history(hist, rows, step, step_stride, row_stride, bos):
    """s [rows, step + 1] = [bos, y_0 .. y_{step-1}] of every row (int64, host)."""
    flat = hist.reshape(-1).cpu().long()
    s = torch.full((rows, step + 1), int(bos), dtype=torch.long)
    if step:
        idx = (torch.arange(rows)[:, None] * row_stride +
               torch.arange(step)[None, :] * step_stride)
        s[:, 1:] = flat[idx]
    return s


def banned(s, ngram):
    """Per row of s [rows, L], the sorted list of tokens the n-gram rule bans."""
    rows, L = s.shape
    if ngram <= 0 or L < ngram:
        return [[] for _ in range(rows)]
    win = s.unfold(1, ngram, 1)                         # rows, L - n + 1, n
    hit = (win[:, :, :ngram - 1] == s[:, L - ngram + 1:][:, None, :]).all(-1)
    return [sorted(set(win[r, :, ngram - 1][hit[r]].tolist())) for r in range(rows)]


def ban_tokens(x, n_valid, hist, *, step_stride, row_stride, bos, step, ngram, min_length, eos):
    from hero_b200 import ops
    if ngram < 0 or min_length < 0 or not 0 <= step < ops.BAN_MAX_HIST \
            or not 1 <= n_valid <= x.shape[1]:
        raise ValueError(f"ban_tokens: ngram {ngram}, min_length {min_length}, step {step}")
    rows = x.shape[0]
    if rows and step > 0 and hist.numel() <= (rows - 1) * row_stride + (step - 1) * step_stride:
        raise ValueError("ban_tokens: the history does not hold every row")
    if ngram == 0 and step >= min_length:
        return
    s = history(hist, rows, step, step_stride, row_stride, bos)
    for r, toks in enumerate(banned(s, ngram)):
        toks = [c for c in toks if 0 <= c < n_valid]
        if toks:
            x[r, torch.tensor(toks, dtype=torch.long, device=x.device)] = -math.inf
    if step < min_length and 0 <= eos < n_valid:
        x[:, eos] = -math.inf


def kept_mask(x, top_k, top_p):
    """bool [rows, n]: the columns of x (already divided by the temperature) that survive top-k
    and top-p."""
    rows, n = x.shape
    key = ord_key(x)
    thr = torch.zeros(rows, dtype=torch.long, device=x.device)
    if 0 < top_k < n:
        thr = torch.sort(key, dim=1, descending=True).values[:, top_k - 1]
    keep = key >= thr[:, None]
    if float(top_p) < 1.0:
        p = float(torch.tensor(float(top_p), dtype=torch.float32))
        mx = x.max(dim=1, keepdim=True).values
        w = torch.floor(torch.exp(x - mx) * 4294967296.0).long()
        w = torch.where(keep, w, torch.zeros_like(w))
        order = torch.sort(key, dim=1, descending=True, stable=True).indices
        cum = torch.cumsum(w.gather(1, order), dim=1)
        for r in range(rows):
            need = max(1, math.ceil(p * float(cum[r, -1])))
            i = int(torch.nonzero(cum[r] >= need)[0])
            keep[r] = key[r] >= key[r, order[r, i]]
    return keep


def uniform_of_hash(h):
    """The fp32 uniform of a 32-bit hash value (int64 tensor)."""
    return ((h >> 9).float() + 0.5) * 2.0 ** -23


def column_hashes(rows, n, seed, step, device=None, row0=0):
    """hash_u32(rkey_r, j) [rows, n] of rows row0 .. row0 + rows - 1 at `step`."""
    r = torch.arange(row0, row0 + rows, dtype=torch.long, device=device)
    rkey = hash_u32(hash_u32(torch.full_like(r, int(seed)), r), step)
    j = torch.arange(n, dtype=torch.long, device=device)
    return hash_u32(rkey[:, None], j[None, :])


def uniforms(rows, n, seed, step, device=None):
    """u [rows, n] fp32 of the draw at `step` (rows 0 .. rows - 1)."""
    return uniform_of_hash(column_hashes(rows, n, seed, step, device))


def largest_uniform(n, seed, step, max_rows=4096, chunk=64):
    """(row, column) of the first row (in order) with a column j < n whose uniform is the largest
    one, 1 - 2^-24 (hash >> 9 == 2^23 - 1), or None within max_rows rows."""
    for row0 in range(0, max_rows, chunk):
        hit = torch.nonzero((column_hashes(chunk, n, seed, step, row0=row0) >> 9) == 2 ** 23 - 1)
        if len(hit):
            return row0 + int(hit[0, 0]), int(hit[0, 1])
    return None


def sample_ref(z, n, *, temperature, top_k, top_p, seed, step):
    """(ids [rows] int64, scores [rows, n] fp32 = x + G over the kept columns, -inf elsewhere)."""
    x = z[:, :n].float() / torch.tensor(float(temperature), dtype=torch.float32)
    keep = kept_mask(x, top_k, top_p)
    g = -torch.log(-torch.log(uniforms(x.shape[0], n, seed, step, x.device)))
    keep = keep & (x > -math.inf)
    v = torch.where(keep, x + g, torch.full_like(x, -math.inf))
    return torch.argmax(v, dim=1), v        # argmax returns the first maximum


def sample_tokens(x, n, ids, *, temperature, top_k, top_p, seed, step):
    from hero_b200 import ops
    if not 1 <= n <= min(ops.SAMPLE_MAX_COLS, x.shape[1]) or not temperature > 0.0 \
            or top_k < 0 or not 0.0 < top_p <= 1.0 or not 0 <= seed < 2 ** 32 or step < 0:
        raise ValueError(f"sample_tokens: n {n}, temperature {temperature}, top_k {top_k}, "
                         f"top_p {top_p}, seed {seed}")
    got, _ = sample_ref(x, n, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                        step=step)
    ids.view(-1)[:x.shape[0]] = got.to(torch.int32)


def install(monkeypatch):
    from tests import fake_beam_ops
    fake_beam_ops.install(monkeypatch)
    from hero_b200 import ops
    for name in ("ban_tokens", "sample_tokens"):
        monkeypatch.setattr(ops, name, globals()[name])
