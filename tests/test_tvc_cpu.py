"""HeroForTvc / TvcGenerator (model/tvc.py) against the unmodified reference on a tiny configuration
(tests/golden/tvc_tiny.npz, written by tools/gen_tvc_golden.py), with hero_b200.ops routed through
tests/fake_tvc_ops.py: the TVC plan, the teacher-forced logits and losses, greedy decoding and the
decoding loop of the evaluation on the host. The CUDA kernel is covered by test_tvc_gpu.py."""
import json

import numpy as np
import pytest
import torch

from oracle import hero_oracle as orc
from tests import fake_tvc_ops
from tests import golden_util as gu


def fixture():
    return gu.load("tvc_tiny.npz")


def tvc_model(tmp_path, tx, lsr=0.1):
    from hero_b200.model import VideoModelConfig
    from hero_b200.tvc import HeroForTvc
    from oracle import gen_golden as gg
    c = json.loads(str(tx["config"]))
    j = gg.model_json(c["hidden"], c["inter"], c["heads"], c["f_layers"], c["c_layers"],
                      c["vocab"])
    j["d_config"] = dict(j["f_config"], num_hidden_layers=c["d_layers"],
                         max_position_embeddings=c["d_max_pos"], type_vocab_size=1)
    path = tmp_path / "tvc.json"
    path.write_text(json.dumps(j))
    model = HeroForTvc(VideoModelConfig(str(path)), vfeat_dim=c["vfeat_dim"],
                       max_frm_seq_len=c["max_frm_seq_len"], lsr=lsr)
    shapes = json.loads(str(tx["state_dict_shapes"]))
    params = {k: s for k, s in shapes.items() if k not in c["buffers"]}
    missing, unexpected = model.load_state_dict(
        orc.seeded_weights(params, seed=c["weight_seed"], std=c["weight_std"]), strict=False)
    assert not unexpected and set(missing) <= set(c["buffers"])
    return model.eval()


def tvc_batch(tx, split="train"):
    b = {k[2:]: torch.from_numpy(v) for k, v in tx.items() if k.startswith("b.")}
    for k in ("clip_ranges", "num_subs", "sub_idx2frame_idx"):
        b[k] = json.loads(str(tx[k]))
    b["clip_ranges"] = tuple(tuple(tuple(r) for r in rs) for rs in b["clip_ranges"])
    if split != "train":
        for k in ("cap_input_ids", "cap_pos_ids", "cap_tgt_ids"):
            del b[k]
    return b


@pytest.mark.parametrize("lsr", [0.1, 0.0])
def test_state_dict_keys_and_shapes_match_reference(tmp_path, lsr):
    tx = fixture()
    ref = json.loads(str(tx["state_dict_shapes" if lsr else "state_dict_shapes_lsr0"]))
    ours = {k: list(v.shape) for k, v in tvc_model(tmp_path, tx, lsr).state_dict().items()}
    assert ours == ref
    assert "decoder.layer.1.intermidiate.dense.weight" in ours and "decoder.tri_mask" in ours


def test_buffers_and_tied_head(tmp_path):
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    tri = model.decoder.tri_mask
    assert tri.shape == (1024, 1024) and tri[0, 1] == -10000.0 and tri[1, 0] == 0.0
    fe = model.v_encoder.f_encoder
    assert fe.lm_head.decoder.weight is fe.embeddings.word_embeddings.weight
    assert model.emb_LayerNorm.eps == 1e-5


@pytest.mark.parametrize("attach", [False, True])
def test_logits_and_losses_match_reference(tmp_path, monkeypatch, attach):
    from hero_b200.plan import attach_plan
    fake_tvc_ops.install(monkeypatch)
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    model0 = tvc_model(tmp_path, tx, lsr=0.0)

    def batch():
        b = tvc_batch(tx)
        return attach_plan(b) if attach else b

    with torch.no_grad():
        logits = model(batch(), compute_loss=False)
        loss = model(batch())
        loss0 = model0(batch())
    ref = tx["logits"]
    assert logits.shape == ref.shape and logits.dtype == torch.float32
    assert np.abs(logits.numpy() - ref).max() <= 2e-2 * np.abs(ref).max()
    for got, want in ((loss, tx["loss_lsr"]), (loss0, tx["loss_ce"])):
        assert got.shape == want.shape
        # per-token losses of ~5 nats: 2e-2 relative (the logits' own error is ~1 % of max |logit|)
        assert (np.abs(got.numpy() - want) <= 2e-2 * np.maximum(np.abs(want), 1.0)).all()
    n_valid = int((tx["b.cap_tgt_ids"] != -1).sum())
    assert loss.shape == (n_valid,) and loss0.numel() == tx["b.cap_tgt_ids"].size


def greedy_agreement(ids, tx, thr):
    """Compare greedy ids with the reference's where the comparison means something: a position
    whose reference top-1 / top-2 logit gap is within `thr` may flip under bf16 rounding, and every
    later position of that caption is then conditioned on a different prefix, so each caption is
    compared up to its first such position. Returns (compared, excluded)."""
    ref, gap = tx["greedy_ids"], tx["greedy_gap"]
    compared = 0
    for r in range(ref.shape[0]):
        low = np.flatnonzero(gap[r] <= thr)
        n = int(low[0]) if low.size else ref.shape[1]
        assert np.array_equal(np.asarray(ids[r][:n]), ref[r][:n]), (r, n)
        compared += n
    return compared, ref.size - compared


def forced_argmax(model, batch, ids, bos):
    """Teacher-forced argmax and top-1 / top-2 gap of the model's own logits with the greedy ids
    as input: the KV-cached decode must pick the same tokens."""
    n, t = ids.shape
    b = dict(batch)
    b["cap_input_ids"] = torch.cat([torch.full((n, 1), bos, dtype=torch.long),
                                    ids[:, :-1].long().cpu()], 1)
    b["cap_pos_ids"] = torch.arange(t).unsqueeze(0)
    with torch.no_grad():
        logits = model(b, compute_loss=False).float().cpu()
    top = logits.topk(2, dim=-1).values
    return logits.argmax(-1), top[..., 0] - top[..., 1]


def test_greedy_ids_match_reference(tmp_path, monkeypatch):
    from hero_b200.tvc import TvcGenerator
    from hero_b200 import synth
    fake_tvc_ops.install(monkeypatch)
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    c = json.loads(str(tx["config"]))
    gen = TvcGenerator(model, c["max_step"], synth.BOS, synth.EOS, fp16=True)
    ids = gen.decode_ids(tvc_batch(tx, "val"))
    assert ids.shape == tx["greedy_ids"].shape and ids.dtype == torch.int32
    # the decode loop equals the teacher-forced pass of the same model on its own output
    am, gap = forced_argmax(model, tvc_batch(tx, "val"), ids, synth.BOS)
    sure = gap > 1e-3
    assert torch.equal(am[sure], ids.long()[sure])
    compared, excluded = greedy_agreement(ids.numpy(), tx, 2 * 2e-2 * np.abs(tx["logits"]).max())
    print(f"greedy ids: {compared} positions compared with the reference, {excluded} after a "
          f"near-tie excluded")
    assert compared > 0
    cut = gen.greedy_decode(tvc_batch(tx, "val"))
    assert cut == [gen.cut_eos(r) for r in ids.tolist()]


def test_tvc_plan_maps_and_empty_segment():
    """Segment s lists the packed clip rows of its frames; the empty segment (st == ed == nframes)
    attends to the zero row alone; decode and teacher-forced ranges."""
    from hero_b200.plan import ReprPlan, TvcPlan
    tx = fixture()
    b = tvc_batch(tx)
    rp = ReprPlan(b)
    p = TvcPlan(b["clip_ranges"], rp)
    cm = b["c_attn_masks"].numpy()
    starts = np.concatenate([[0], np.cumsum(cm.sum(1))])
    segs = [(v, st, ed) for v, rs in enumerate(b["clip_ranges"]) for st, ed in rs]
    assert p.n_seg == len(segs) == b["cap_input_ids"].shape[0]
    assert p.seg_src[-1] == -1 and p.n_rows == p.seg_src.size
    for i, (v, st, ed) in enumerate(segs):
        if st == ed:
            assert (p.kv_off[i], p.kv_len[i]) == (p.n_rows - 1, 1)
            continue
        rows = p.seg_src[p.kv_off[i]:p.kv_off[i] + p.kv_len[i]]
        assert rows.tolist() == list(range(starts[v] + st, starts[v] + ed))
    assert (p.seg_len == b["cap_attn_mask"].sum(1).numpy()).all()
    d = p.decode_arrays(5)
    assert d["self_off"].tolist() == [5 * i for i in range(p.n_seg)]
    assert d["step_len"].reshape(5, -1)[3].tolist() == [4] * p.n_seg
    assert d["step_pos"].reshape(5, -1)[3].tolist() == [3] * p.n_seg
    f = p.forced_arrays(4)
    assert f["tf_self_off"][4:8].tolist() == [4] * 4 and f["tf_self_len"][:4].tolist() == [1, 2, 3, 4]
    assert f["tf_kv_len"][:4].tolist() == [p.kv_len[0]] * 4


def test_tvc_plan_rejects_bad_segments():
    from hero_b200.plan import ReprPlan, TvcPlan
    b = tvc_batch(fixture())
    rp = ReprPlan(b)
    nfr = int(b["c_attn_masks"][0].sum())
    bad = ((0, nfr + 1),) + b["clip_ranges"][0][1:]
    with pytest.raises(ValueError, match="outside"):
        TvcPlan((bad,) + b["clip_ranges"][1:], rp)
    empty = tuple(tuple((int(m.sum()), int(m.sum())) for _ in rs)
                  for m, rs in zip(b["c_attn_masks"], b["clip_ranges"]))
    with pytest.raises(ValueError, match="empty"):
        TvcPlan(empty, rp)


def test_empty_segment_attends_to_the_value_bias(tmp_path, monkeypatch):
    """The zero row's cross-attention K / V are the biases, so an empty segment's cross-attention
    output is exactly b_v, as the reference's uniformly masked zero padding gives."""
    fake_tvc_ops.install(monkeypatch)
    from hero_b200 import ops
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    b = tvc_batch(tx)
    with torch.no_grad():
        y, plan = model.encode(b)
        tdev = plan.to("cpu")
        enc = model._gather_segments(y, plan, tdev)
        assert (enc[-1] == 0).all()
        flat, w = model._weights(torch.device("cpu"))
        kv = model._cross_kv(w, enc)[0]
    H = enc.shape[1]
    q = torch.randn(plan.n_seg, H).to(torch.bfloat16)
    out = torch.empty(plan.n_seg, H, dtype=torch.bfloat16)
    ops.dec_attn_fwd(q, kv[:, :H], kv[:, H:], tdev.kv_off, tdev.kv_len, out, heads=2,
                     max_kv_len=plan.max_kv)
    bv = model.decoder.layer[0].dec_enc_attention.value.bias
    i = int(np.flatnonzero(plan.seg_len == 0)[0])
    assert torch.equal(out[i].float(), bv.to(torch.bfloat16).float())


def test_forward_refuses_training(tmp_path, monkeypatch):
    fake_tvc_ops.install(monkeypatch)
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    with pytest.raises(NotImplementedError, match="decoder training is not on the CUDA path"):
        model(tvc_batch(tx))                         # grad enabled, parameters require it
    model.train()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="training"):
        model(tvc_batch(tx), compute_loss=False)


def test_max_step_bounds(tmp_path, monkeypatch):
    from hero_b200.tvc import TvcGenerator
    fake_tvc_ops.install(monkeypatch)
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    for bad in (0, 1024):
        with pytest.raises(ValueError, match="max_step"):
            TvcGenerator(model, bad, 0, 2, False).greedy_decode(tvc_batch(tx, "val"))


def test_dec_attn_bounds_raise_before_launch():
    from hero_b200 import ops
    z = torch.zeros(2, 128, dtype=torch.bfloat16)
    i = torch.zeros(2, dtype=torch.int32)
    for kw in (dict(max_kv_len=1025), dict(max_kv_len=4, min_kv_len=0),
               dict(max_kv_len=4, head_dim=32)):
        with pytest.raises(ValueError, match="dec_attn_fwd"):
            ops.dec_attn_fwd(z, z, z, i, i, z, heads=2, **kw)


class _Stub:
    """Tokenizer stand-in: ids -> 'w<id>' tokens, joined with spaces."""

    def convert_ids_to_tokens(self, ids):
        return [f"w{i}" for i in ids]

    def convert_tokens_to_string(self, toks):
        return " ".join(toks)


def test_decode_tvc_records(tmp_path, monkeypatch):
    """evalpass.decode_tvc follows inf_tvc.py:83-98: one record per caption segment, in batch
    order, with the greedy caption of TvcGenerator decoded by the tokenizer."""
    from hero_b200 import evalpass, synth
    from hero_b200.tvc import TvcGenerator
    fake_tvc_ops.install(monkeypatch)
    tx = fixture()
    model = tvc_model(tmp_path, tx)
    c = json.loads(str(tx["config"]))
    vb = synth.syn_tvc_batch(**c["batch_args"], split="val")
    loader = [vb, dict(vb)]
    recs = evalpass.decode_tvc(model, loader, max_step=c["max_step"], bos=synth.BOS,
                               eos=synth.EOS, tokenizer=_Stub())
    gen = TvcGenerator(model, c["max_step"], synth.BOS, synth.EOS, False)
    want = gen.greedy_decode(vb)
    assert len(recs) == 2 * len(vb["clip_ids"])
    for r, vid, cid, ts, ids in zip(recs, vb["vid_names"] * 2, vb["clip_ids"] * 2,
                                    vb["all_ts"] * 2, want * 2):
        assert set(r) == {"vid_name", "clip_id", "ts", "descs"}
        assert (r["vid_name"], r["clip_id"], r["ts"]) == (vid, cid, ts)
        assert r["descs"] == [{"desc": " ".join(f"w{i}" for i in ids)}]
