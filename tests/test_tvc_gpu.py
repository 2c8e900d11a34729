"""TVC captioning on the H100: the decoder-attention kernel (csrc/decode.cu) against the torch
restatement of its range contract, rank_topk(k=1) as the greedy argmax, HeroForTvc against the
reference's outputs (tests/golden/tvc_tiny.npz) and, at real dimensions, against the reference
module staged under oracle/_ref, and greedy decoding without host synchronisation."""
import json

import numpy as np
import pytest
import torch

from tests import fake_tvc_ops
from tests import test_tvc_cpu as cpu
from tests import test_videoqa_gpu as qa_gpu

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
BF16 = torch.bfloat16


def _ranges(kind, rows, n_kv, gen):
    """(kv_off, kv_len) of the three uses of the kernel."""
    if kind == "causal":          # rows = captions x positions, keys 0..t of the caption
        L = 37
        n = torch.arange(rows) // L
        t = torch.arange(rows) % L
        return n * L, t + 1
    if kind == "decode":          # one query per caption against a cache of T rows per caption
        T = 30
        return torch.arange(rows) * T, torch.randint(1, T + 1, (rows,), generator=gen)
    if kind == "cross":           # ragged segment ranges, one of length 1024, some of length 1
        lens = torch.randint(1, 120, (rows,), generator=gen)
        lens[0], lens[1] = 1024, 1
        off = torch.randint(0, n_kv - 1024, (rows,), generator=gen)
        return off, lens
    raise ValueError(kind)


@pytest.mark.parametrize("kind,rows,heads", [("causal", 74, 12), ("decode", 33, 12),
                                             ("cross", 40, 2)])
def test_dec_attn_matches_torch(kind, rows, heads):
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(3)
    H = heads * 64
    n_kv = 2048 if kind == "cross" else rows * 37 + 64
    # q / k / v as strided column blocks of one QKV buffer, as the decoder passes them
    qkv = torch.randn(max(n_kv, rows), 3 * H, generator=gen).to(BF16).to(DEV)
    q, k, v = qkv[:rows, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    off, lens = _ranges(kind, rows, n_kv, gen)
    off_d, len_d = off.int().to(DEV), lens.int().to(DEV)
    out = torch.full((rows, H), float("nan"), dtype=BF16, device=DEV)
    ops.dec_attn_fwd(q, k, v, off_d, len_d, out, heads=heads, max_kv_len=int(lens.max()))
    torch.cuda.synchronize()
    ref = fake_tvc_ops.dec_attn_ref(q, k, v, off_d, len_d, heads)
    assert not torch.isnan(out).any()
    torch.testing.assert_close(out.float(), ref, rtol=8e-3, atol=2e-3)
    one = (lens == 1).nonzero().view(-1)
    for i in one.tolist():            # a single key returns its value row exactly
        assert torch.equal(out[i], v[int(off[i])])


def test_dec_attn_out_of_bounds_raise_before_launch():
    from hero_b200 import ops
    z = torch.full((4, 128), float("nan"), dtype=BF16, device=DEV)
    i = torch.ones(4, dtype=torch.int32, device=DEV)
    for kw in (dict(max_kv_len=1025), dict(max_kv_len=4, min_kv_len=0),
               dict(max_kv_len=4, head_dim=32)):
        with pytest.raises(ValueError, match="dec_attn_fwd"):
            ops.dec_attn_fwd(z, z, z, i, i, z, heads=2, **kw)
    torch.cuda.synchronize()
    assert torch.isnan(z).all()          # nothing was launched


def test_rank_topk_k1_is_argmax_with_ties_to_the_lower_column():
    from hero_b200 import ops
    gen = torch.Generator().manual_seed(0)
    V = 50272
    x = torch.randn(48, V + 16, generator=gen).to(DEV)
    x[3, 100] = x[3, 40000] = 50.0                  # exact ties: the lower column wins
    x[7, 0] = x[7, V - 1] = 60.0
    x[9, V - 1] = 70.0                              # the last real column
    x[11, V + 3] = 1e9                              # beyond n: not a candidate
    idx = torch.empty(48, 1, dtype=torch.int32, device=DEV)
    val = torch.empty(48, 1, device=DEV)
    ops.rank_topk(x, V, 1, val, idx)
    want = torch.argmax(x[:, :V], dim=1)
    assert torch.equal(idx.view(-1).long(), want)
    assert idx[3, 0] == 100 and idx[7, 0] == 0 and idx[9, 0] == V - 1


def test_model_matches_reference_fixture(tmp_path):
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    from hero_b200.tvc import TvcGenerator
    tx = cpu.fixture()
    model = cpu.tvc_model(tmp_path, tx).to(DEV)
    model0 = cpu.tvc_model(tmp_path, tx, lsr=0.0).to(DEV)

    def batch(split="train"):
        return synth.to_device(attach_plan(cpu.tvc_batch(tx, split)), DEV)

    with torch.no_grad():
        logits = model(batch(), compute_loss=False).cpu()
        loss, loss0 = model(batch()).cpu(), model0(batch()).cpu()
    ref = tx["logits"]
    err = float(np.abs(logits.numpy() - ref).max())
    bound = 2e-2 * float(np.abs(ref).max())
    print(f"tiny fixture: logits max error {err:.4f} (bound {bound:.4f})")
    assert err <= bound
    for got, want in ((loss, tx["loss_lsr"]), (loss0, tx["loss_ce"])):
        assert got.shape == want.shape
        assert (np.abs(got.numpy() - want) <= 2e-2 * np.maximum(np.abs(want), 1.0)).all()
    c = json.loads(str(tx["config"]))
    gen = TvcGenerator(model, c["max_step"], synth.BOS, synth.EOS, fp16=True)
    ids = gen.decode_ids(batch("val"))
    am, gap = cpu.forced_argmax(model, batch("val"), ids, synth.BOS)
    sure = gap > 1e-3
    assert torch.equal(am[sure], ids.long()[sure])
    compared, excluded = cpu.greedy_agreement(ids.numpy(), tx, 2 * bound)
    print(f"greedy ids: {compared} positions compared with the reference, {excluded} after a "
          f"near-tie (gap <= {2 * bound:.3f}) excluded")
    assert compared > 0


def test_greedy_decode_makes_one_copy_and_no_sync():
    from torch.profiler import ProfilerActivity, profile
    from hero_b200 import synth
    from hero_b200.plan import attach_plan
    from hero_b200.tvc import TvcGenerator
    model, _ = _tvc_model(layers=(2, 2, 2), hidden=256, heads=4, vocab=1000)
    model = model.to(DEV).eval()
    b = attach_plan(synth.syn_tvc_batch(n_videos=8, seed=4, vfeat_dim=64, vocab=1000,
                                        split="val"))
    gen = TvcGenerator(model, 30, synth.BOS, synth.EOS, fp16=False)
    db = synth.to_device(b, DEV)
    first = gen.greedy_decode(db)                   # warm-up (allocations, weight mirror)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gen.greedy_decode(synth.to_device(b, DEV))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert out == first and len(out) == len(b["clip_ids"])
    db = synth.to_device(b, DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gen.greedy_decode(db)
        torch.cuda.synchronize()
    d2h = [e for e in prof.events() if "Memcpy DtoH" in e.name]
    assert len(d2h) == 1, [e.name for e in d2h]


def _tvc_model(layers=(6, 3, 2), hidden=768, heads=12, vocab=50272, seed=0):
    import tempfile
    from hero_b200.model import VideoModelConfig
    from hero_b200.tvc import HeroForTvc
    from oracle import gen_golden as gg
    f_l, c_l, d_l = layers
    j = gg.model_json(hidden, 4 * hidden, heads, f_l, c_l, vocab)
    j["d_config"] = dict(j["f_config"], num_hidden_layers=d_l, max_position_embeddings=1024,
                         type_vocab_size=1)
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as f:
        json.dump(j, f)
        path = f.name
    torch.manual_seed(seed)
    vfeat = 4352 if hidden == 768 else 64
    return HeroForTvc(VideoModelConfig(path), vfeat_dim=vfeat, max_frm_seq_len=100), path


def test_real_dimensions_match_staged_reference():
    """6 + 3 encoder layers, 2 decoder layers, H 768, vocabulary 50 272, eval mode: teacher-forced
    logits against the reference's HeroForTvc in fp32 on the same GPU, with the same reference under
    torch bf16 autocast as the yardstick (<= 3e-2 relative, or <= 1.5x its error); the argmax must
    agree wherever the reference's top-1 / top-2 gap exceeds twice our error."""
    VideoModelConfig, _ = qa_gpu._reference_module()
    from model.tvc import HeroForTvc as RefTvc
    from hero_b200 import synth
    model, path = _tvc_model(seed=3)
    ref = RefTvc(VideoModelConfig(path), vfeat_dim=4352, max_frm_seq_len=100)
    ref.load_state_dict(model.state_dict())
    model, ref = model.to(DEV).eval(), ref.to(DEV).eval()
    hb = synth.syn_tvc_batch(n_videos=4, seed=9, vocab=50265)
    with torch.no_grad():
        lo = model(synth.to_device(hb, DEV), compute_loss=False).float()
        lr = ref(synth.to_device(hb, DEV), compute_loss=False).float()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            lb = ref(synth.to_device(hb, DEV), compute_loss=False).float()
    scale = float(lr.abs().max())
    ours, bf16 = float((lo - lr).abs().max()) / scale, float((lb - lr).abs().max()) / scale
    print(f"real dimensions: logits rel err vs fp32 reference: ours {ours:.4f}, "
          f"reference bf16 {bf16:.4f}")
    assert ours <= 3e-2 or ours <= 1.5 * bf16, (ours, bf16)
    top = lr.topk(2, dim=-1).values
    gap = top[..., 0] - top[..., 1]
    sure = gap > 2 * ours * scale
    agree = lo.argmax(-1) == lr.argmax(-1)
    print(f"teacher-forced argmax: {int(sure.sum())} of {sure.numel()} positions past the gap "
          f"bound, {int(agree.sum())} agree overall")
    assert bool(agree[sure].all())
