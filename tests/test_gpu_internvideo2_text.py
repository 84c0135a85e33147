"""InternVideo2 text tower on the GPU: cb_attention_masked_f16 against oracle/attention.py on each sequence's valid keys, the post-LN
LayerNorm and the embedding gather against torch, cb_iv2_text_* against the reference's BertModel golden (depth 2) and the float32
oracle at full depth, bitwise independence of a text's embedding from its neighbours, its slot and the padded length, the error codes,
and InternVideo2FrameCreationStage -> InternVideo2EmbeddingStage(texts_to_verify=...)."""

from __future__ import annotations

import os
import uuid

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, golden_json, load_golden
from gpu_helpers import ctx  # noqa: F401
from oracle import attention as A
from oracle import internvideo2_text as O

pytestmark = pytest.mark.gpu

HD = 64
PAD = 3
SENTINEL = -7777.0
VOCAB = GOLDEN / "bert_vocab_synth.txt"


# ------------------------------------------------------------------------------------------------------------ masked attention
def _masked(ctx, qkv: torch.Tensor, heads: int, lengths) -> torch.Tensor:
    """cb_attention_masked_f16 on qkv [n][T][3 * hidden] between NaN rows, writing into a sentinel-filled buffer; asserts nothing outside
    the output was written."""
    from cosmos_curate_b200.runtime import _stream_ptr, check

    n, t, three_hidden = qkv.shape
    hidden, rows = three_hidden // 3, n * t
    src = torch.full((rows + 2 * PAD, three_hidden), float("nan"), dtype=torch.float16, device="cuda")
    src[PAD : PAD + rows] = qkv.reshape(rows, three_hidden)
    dst = torch.full((rows + 2 * PAD, hidden), SENTINEL, dtype=torch.float16, device="cuda")
    lens = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    check(ctx.lib.cb_attention_masked_f16(ctx.h, src[PAD:].data_ptr(), dst[PAD:].data_ptr(), n, t, heads, hidden // heads, lens.data_ptr(),
                                          _stream_ptr()), "cb_attention_masked_f16", ctx.h)  # fmt: skip
    torch.cuda.synchronize()
    assert (dst[:PAD] == SENTINEL).all() and (dst[PAD + rows :] == SENTINEL).all(), "rows outside [n*T][hidden] were written"
    return dst[PAD : PAD + rows].view(n, t, hidden)


def _pad(parts, t: int, fill: str, seed: int = 0) -> torch.Tensor:
    """Sequences [len_i][3 * hidden] -> [n][T][3 * hidden]; rows past each length hold `fill`: "poison" (Inf / NaN / -Inf) or "random"."""
    three_hidden = parts[0].shape[-1]
    out = torch.empty(len(parts), t, three_hidden, dtype=torch.float16)
    g = torch.Generator().manual_seed(seed)
    if fill == "poison":
        out[:] = torch.tensor([float("inf"), float("nan"), float("-inf")], dtype=torch.float16)[torch.arange(three_hidden) % 3]
    else:
        out[:] = (torch.randn(len(parts), t, three_hidden, generator=g) * 3).half()
    for i, p in enumerate(parts):
        out[i, : p.shape[0]] = p
    return out.cuda()


def _bitwise(got, want, what):
    bad = (got.contiguous().view(torch.int16) != want.contiguous().view(torch.int16)).nonzero()
    assert len(bad) == 0, f"{what}: {len(bad)} elements differ, first at {bad[0].tolist()}"


MASK_T = [1, 16, 17, 40, 64, 129, 257, 352]


def _lengths(t):
    return sorted({x for x in (1, 2, 15, 16, 17, 31, 32, 33, 40, t) if x <= t})


@pytest.fixture(scope="module")
def worst():
    w = {"masked": 0.0}
    yield w
    print(f"\nattention masked: worst err/bound {w['masked']:.3f}")


@pytest.mark.parametrize("t", MASK_T)
def test_masked_attention_sweep(ctx, monkeypatch, worst, t):
    """Exact selection / uniform answers and the rounding bound on each sequence's own keys; padding rows of Inf and NaN change nothing;
    each sequence equals cb_attention_f16's mma.sync kernel on the unpadded sequence bit for bit; rows past the length are zeros."""
    from cosmos_curate_b200.runtime import _stream_ptr

    heads, lens = 2, _lengths(t)
    n = len(lens)
    # selection: row i of (sequence, head) is V[pi(i)], pi over the sequence's own keys
    sel = [A.selection_inputs(1, ln, heads, HD, seed=t * 100 + ln) for ln in lens]
    out = _masked(ctx, _pad([q[0] for q, _ in sel], t, "poison"), heads, lens)
    for b, ((qkv, pi), ln) in enumerate(zip(sel, lens)):
        v = A.split_heads(qkv, heads)[2]
        _bitwise(out[b, :ln], A.merge_heads(torch.gather(v, 2, pi[..., None].expand(-1, -1, -1, HD)))[0].cuda(), f"selection T={t} len={ln}")
        assert (out[b, ln:] == 0).all(), f"rows past length {ln} are not zero"
    # uniform: the per-sequence constant
    uni = [A.uniform_inputs(1, ln, heads, HD, seed=t + ln) for ln in lens]
    out = _masked(ctx, _pad([q[0] for q, _ in uni], t, "poison"), heads, lens)
    for b, ((_, c), ln) in enumerate(zip(uni, lens)):
        _bitwise(out[b, :ln], A.merge_heads(c[:, :, None, :].expand(1, heads, ln, HD)).half()[0].cuda(), f"uniform T={t} len={ln}")
    # random: within the bound of the truncated sequence; poison vs random padding bitwise; vs the unpadded sequence on cb_attention_f16
    monkeypatch.setenv("CB_ATTN_KERNEL", "mma")
    for kind in ("normal", "sharp", "large", "ties"):
        parts = [A.random_inputs(1, ln, heads, HD, seed=7 * t + ln, kind=kind)[0] for ln in lens]
        poisoned = _masked(ctx, _pad(parts, t, "poison"), heads, lens)
        clean = _masked(ctx, _pad(parts, t, "random", seed=t), heads, lens)
        for b, (p, ln) in enumerate(zip(parts, lens)):
            assert torch.isfinite(poisoned[b]).all()
            _bitwise(poisoned[b, :ln], clean[b, :ln], f"{kind} T={t} len={ln}: poisoned vs random padding")
            ref, s_abs = A.reference(p[None].cuda(), heads)
            ratio = ((poisoned[b : b + 1, :ln].double() - ref).abs() / A.bound(ref, s_abs, p[None].cuda(), heads)).max().item()
            worst["masked"] = max(worst["masked"], ratio)
            assert ratio <= 1.0, f"{kind} T={t} len={ln}: err/bound {ratio:.3f}"
            p_dev = p.cuda()
            alone = torch.empty(1, ln, heads * HD, dtype=torch.float16, device="cuda")
            assert ctx.lib.cb_attention_f16(ctx.h, p_dev.data_ptr(), alone.data_ptr(), 1, ln, heads, HD, _stream_ptr()) == 0
            torch.cuda.synchronize()
            _bitwise(poisoned[b, :ln], alone[0], f"{kind} T={t} len={ln}: vs the unpadded sequence")


@pytest.mark.parametrize("t", MASK_T)
def test_masked_attention_full_lengths_is_cb_attention_f16(ctx, monkeypatch, t):
    """Every length == T: bitwise cb_attention_f16 (its mma.sync kernel; for 129..257 tokens forced with CB_ATTN_KERNEL=mma)."""
    qkv = A.random_inputs(3, t, 4, HD, seed=t, kind="sharp").cuda()
    got = _masked(ctx, qkv, 4, [t] * 3)
    for force in (True, False):
        if not force and A.path_of(t, HD) != "mma64_resident":
            continue
        if force:
            monkeypatch.setenv("CB_ATTN_KERNEL", "mma")
        else:
            monkeypatch.delenv("CB_ATTN_KERNEL", raising=False)
        _bitwise(got, ctx.attention(qkv, 4), f"T={t} force_mma={force}")


@pytest.mark.parametrize(("t", "hd"), [(40, 32), (40, 80), (40, 88), (353, 64), (512, 64)])
def test_masked_attention_unsupported(ctx, t, hd):
    from cosmos_curate_b200.runtime import _stream_ptr

    heads = 2
    qkv = torch.zeros(t, 3 * heads * hd, dtype=torch.float16, device="cuda")
    out = torch.full((t, heads * hd), SENTINEL, dtype=torch.float16, device="cuda")
    lens = torch.tensor([t], dtype=torch.int32, device="cuda")
    assert ctx.lib.cb_attention_masked_f16(ctx.h, qkv.data_ptr(), out.data_ptr(), 1, t, heads, hd, lens.data_ptr(), _stream_ptr()) == -3
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()
    assert ctx.lib.cb_attention_masked_f16(ctx.h, qkv.data_ptr(), out.data_ptr(), 0, 40, heads, 64, lens.data_ptr(), _stream_ptr()) == 0


# ------------------------------------------------------------------------------------------------------- LayerNorm, gather
@pytest.mark.parametrize(("rows", "d"), [(1, 1024), (333, 1024), (40, 768), (17, 1536)])
def test_layernorm_post_in_place_and_fp16_copy(ctx, rows, d):
    g = torch.Generator(device="cuda").manual_seed(rows + d)
    h = torch.randn(rows, d, device="cuda", generator=g) * 3 + 1
    gamma = 1 + 0.2 * torch.rand(d, device="cuda", generator=g)
    beta = 0.1 * torch.randn(d, device="cuda", generator=g)
    want = F.layer_norm(h.double(), (d,), gamma.double(), beta.double(), 1e-12)
    x = h.clone()
    y = ctx.layernorm_post_(x, gamma, beta, 1e-12)
    assert (x.double() - want).abs().max().item() <= 2e-5
    assert torch.equal(y, x.half())  # the fp16 copy is the fp32 result rounded
    # the same statistics as cb_layernorm_f16
    assert torch.equal(y, ctx.layernorm(h, gamma, beta, 1e-12))


def test_text_embed_gather(ctx):
    g = torch.Generator(device="cuda").manual_seed(5)
    vocab, max_pos, d, n, L = 300, 64, 1024, 3, 40
    word, pos, typ = (torch.randn(s, device="cuda", generator=g) for s in ((vocab, d), (max_pos, d), (d,)))
    ids = torch.randint(0, vocab, (n, L), device="cuda", generator=g, dtype=torch.int32)
    got = ctx.text_embed(ids, word, pos, typ)
    assert torch.equal(got, (word[ids.long()] + typ) + pos[:L])


# ------------------------------------------------------------------------------------------------------------------- tower
def _errors(got: np.ndarray, want: np.ndarray):
    cos = (got * want).sum(-1) / (np.linalg.norm(got, axis=-1) * np.linalg.norm(want, axis=-1))
    return float(1 - cos.min()), float(np.abs(got - want).max())


def test_tower_matches_the_reference_bert(ctx):
    """cb_iv2_text_forward on the golden batch (the reference's BertModel in float32 at depth 2, 1024 wide): 1 - cosine <= 1e-6, max-abs
    <= 1e-3; the reference's own bf16 run is printed beside it."""
    from cosmos_curate_b200.runtime import Iv2TextTower

    g = load_golden("internvideo2_text_ref.npz")
    meta = golden_json(g, "meta")
    cfg = O.IV2_TEXT.with_(layers=meta["depth"], vocab=meta["vocab"])
    tower = Iv2TextTower(ctx, cfg.to_dict(), O.random_weights(cfg, meta["seed"]), max_texts=8, max_len=40)
    got = tower.forward(g["ids"], g["lengths"]).cpu().numpy()
    tower.close()
    e_cos, e_abs = _errors(got, g["emb"])
    b_cos, b_abs = _errors(g["emb_bf16"], g["emb"])
    print(f"\ntext tower vs reference (depth 2): 1-cos {e_cos:.2e} max-abs {e_abs:.2e} | reference bf16: 1-cos {b_cos:.2e} max-abs {b_abs:.2e}")
    assert e_cos <= 1e-6 and e_abs <= 1e-3


@pytest.fixture(scope="module")
def full_tower(ctx):
    from cosmos_curate_b200.runtime import Iv2TextTower

    cfg = O.IV2_TEXT
    w = O.random_weights(cfg, seed=31)
    tower = Iv2TextTower(ctx, cfg.to_dict(), w, max_texts=64, max_len=64)
    yield cfg, w, tower
    tower.close()


def _random_texts(n, L, seed, vocab=30522):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(2, L + 1, n).astype(np.int32)
    ids = np.zeros((n, L), np.int32)
    for i, ln in enumerate(lengths):
        ids[i, 0], ids[i, 1 : ln - 1], ids[i, ln - 1] = 101, rng.integers(999, vocab, ln - 2), 102
    return ids, lengths


def test_tower_full_depth_against_the_oracle(ctx, full_tower):
    """19 layers at 1024 wide on seeded weights, texts of several lengths: fp16 GEMM operands vs the float32 oracle."""
    cfg, w, tower = full_tower
    ids, lengths = _random_texts(6, 40, seed=1)
    lengths[0], lengths[1] = 40, 2
    ids[0, 39], ids[1, 1] = 102, 102
    got = tower.forward(ids, lengths).cpu().numpy()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            want = O.forward(cfg, w, ids, lengths, device="cuda").cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    for i in range(len(ids)):
        e_cos, e_abs = _errors(got[i : i + 1], want[i : i + 1])
        print(f"\nfull depth text {i} (length {lengths[i]}): 1-cos {e_cos:.2e} max-abs {e_abs:.2e}")
    e_cos, e_abs = _errors(got, want)
    assert np.allclose(np.linalg.norm(got, axis=1), 1, atol=1e-6)
    assert e_cos <= 1e-5 and e_abs <= 1e-3


def test_tower_is_bitwise_independent_of_neighbours_slot_and_padding(ctx, full_tower):
    """Each text alone at its own length, in a batch at L = 40, at L = 64, in reverse order and among 200 texts (four chunks, other GEMM
    tiles): the same bits."""
    _, _, tower = full_tower
    ids, lengths = _random_texts(200, 40, seed=2)
    batch = tower.forward(ids, lengths).cpu().numpy()
    for i in range(0, 200, 37):
        alone = tower.forward(ids[i : i + 1, : lengths[i]], lengths[i : i + 1]).cpu().numpy()
        assert np.array_equal(alone[0], batch[i]), i
    few = tower.forward(ids[:5], lengths[:5]).cpu().numpy()
    assert np.array_equal(few, batch[:5])
    rev = tower.forward(ids[:5][::-1], lengths[:5][::-1]).cpu().numpy()
    assert np.array_equal(rev[::-1], batch[:5])
    wide = np.full((5, 64), 7, np.int32)  # other token ids in the padding
    wide[:, :40] = ids[:5]
    assert np.array_equal(tower.forward(wide, lengths[:5]).cpu().numpy(), batch[:5])


def test_tower_invalid_inputs(ctx, full_tower):
    from cosmos_curate_b200._lib import CurateB200Error

    _, _, tower = full_tower
    ids, lengths = _random_texts(3, 40, seed=3)
    for bad_ids, bad_len in ((np.where(np.arange(40) == 5, 30522, ids), lengths), (np.where(np.arange(40) == 0, -1, ids), lengths),
                             (ids, np.array([3, 0, 5], np.int32)), (ids, np.array([3, 41, 5], np.int32))):  # fmt: skip
        with pytest.raises(CurateB200Error) as e:
            tower.forward(bad_ids, bad_len)
        assert e.value.code == -7  # CB_ERR_INVALID
    with pytest.raises(CurateB200Error) as e:
        tower.forward(np.zeros((1, 513), np.int32), np.array([3], np.int32))
    assert e.value.code == -7
    with pytest.raises(CurateB200Error) as e:
        tower.forward(np.zeros((1, 65), np.int32), np.array([3], np.int32))  # past the workspace's max_len
    assert e.value.code == -2
    assert tower.forward(ids, lengths).shape == (3, 512)  # the handle still works


# ------------------------------------------------------------------------------------------------------------ end to end
def test_frame_creation_then_embedding_stage_with_texts(ctx):
    """InternVideo2FrameCreationStage -> InternVideo2EmbeddingStage(texts_to_verify=...) on seeded weights: each clip's match is the
    oracle's choice and probability.  Each clip gets its own two texts, picked with the oracle from 400 random captions: the best and the
    worst, at least 5 logits apart, so that no near-tie can flip the choice and the probability (>= 0.993) is insensitive to rounding."""
    from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
    from cosmos_curate_b200.models.bert_tokenizer import BertTokenizer
    from cosmos_curate_b200.models.internvideo2 import IV2_1B_CFG, IV2_TEXT_CFG, InternVideo2MultiModality, seeded_text_weights, seeded_weights
    from cosmos_curate_b200.models.internvideo2_frames import InternVideo2FrameFormulator
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage, InternVideo2FrameCreationStage
    from oracle import internvideo2 as V
    from tools import synth_h264

    datas = [(GOLDEN / "sintel_clip_10s.mp4").read_bytes(), synth_h264.make_clip(640, 360, 30, 3.0, seed=5, gop=30, pan=(2, 1)), None]
    clips = [Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, 3.0), encoded_data=d) for d in datas]
    frames_stage = InternVideo2FrameCreationStage(target_fps=2.0, source="nvdec", model=InternVideo2FrameFormulator(num_frames=4))
    frames_stage.stage_setup()
    frames_stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips))])
    tubes = np.concatenate([clips[i].intern_video_2_frames.resolve() for i in (0, 1)])

    tok = BertTokenizer.from_file(VOCAB)
    vcfg, tcfg = dict(IV2_1B_CFG, layers=2), dict(IV2_TEXT_CFG, layers=2, vocab=len(tok.vocab))
    rng = np.random.default_rng(11)
    words = [w for w in tok.vocab if not w.startswith(("[", "##"))]
    pool = [" ".join(rng.choice(words, rng.integers(1, 40))) for _ in range(400)]
    with torch.no_grad():  # the oracle's clip and text embeddings
        v = V.forward(V.IV2_1B.with_(layers=2), seeded_weights(vcfg, 7), torch.from_numpy(tubes), device="cuda").cpu().numpy()
        ids, lengths = tok(pool, 40)
        t = O.forward(O.IV2_TEXT.with_(layers=2, vocab=len(tok.vocab)), seeded_text_weights(tcfg, 7), ids, lengths, device="cuda").cpu().numpy()
    logits = (100.0 * v @ t.T).astype(np.float32)  # [2][pool]

    model = InternVideo2MultiModality(seed=7, config=vcfg, text_config=tcfg, vocab_file=VOCAB, max_clips=8)
    for i in (0, 1):
        order = np.argsort(-logits[i], kind="stable")
        chosen = [int(order[-1]), int(order[0])]  # the worst caption, then the best
        texts = [pool[j] for j in chosen]
        gap = logits[i, order[0]] - logits[i, order[-1]]
        probs = torch.from_numpy(logits[i, chosen]).softmax(-1).numpy()
        stage = InternVideo2EmbeddingStage(batch_size=8, model=model, texts_to_verify=texts)
        stage.stage_setup()
        stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=[clips[i], clips[2]]))])
        text, p = clips[i].intern_video_2_text_match
        print(f"\nclip {i}: chose text {texts.index(text)} p={p:.6f} | oracle: text 1 p={probs.max():.6f}, lead {gap:.1f} logits")
        assert gap >= 5.0
        assert text == texts[1] and abs(p - float(probs[1])) <= 1e-4
    assert clips[2].intern_video_2_embedding is None and clips[2].intern_video_2_text_match is None
    # the model's text embeddings against the oracle's
    got = model.encode_texts(pool[:16])
    e_cos, e_abs = _errors(got, t[:16])
    assert e_cos <= 1e-6 and e_abs <= 1e-3
    assert np.array_equal(model.get_text_embedding(pool[3]).numpy()[0], got[3])


@pytest.mark.skipif(not (os.environ.get("CURATE_B200_IV2_CHECKPOINT") and os.environ.get("CURATE_B200_BERT_VOCAB")),
                    reason="set CURATE_B200_IV2_CHECKPOINT (InternVideo2-stage2_1b-224p-f4.pt) and CURATE_B200_BERT_VOCAB (bert-large-uncased vocab.txt)")  # fmt: skip
def test_reference_real_weight_text_tower(ctx):
    """The real checkpoint's text tower through the model class vs oracle/internvideo2_text.py in float32 on the same weights."""
    from cosmos_curate_b200.models.internvideo2 import IV2_TEXT_CFG, InternVideo2MultiModality, load_text_checkpoint

    model = InternVideo2MultiModality(checkpoint=os.environ["CURATE_B200_IV2_CHECKPOINT"], vocab_file=os.environ["CURATE_B200_BERT_VOCAB"])
    texts = ["a dog running on the beach", "A man rides a bicycle down a busy city street at night.", "cooking pasta in a small kitchen", "雪"]
    got = model.encode_texts(texts)
    ids, lengths = model.tokenizer(texts, 40)
    w = load_text_checkpoint(os.environ["CURATE_B200_IV2_CHECKPOINT"], IV2_TEXT_CFG)
    with torch.no_grad():
        want = O.forward(O.IV2_TEXT, w, ids, lengths, device="cuda").cpu().numpy()
    e_cos, e_abs = _errors(got, want)
    print(f"\nreal text tower: 1-cos {e_cos:.2e} max-abs {e_abs:.2e}")
    assert e_cos <= 1e-5 and e_abs <= 1e-3
