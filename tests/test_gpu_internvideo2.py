"""InternVideo2 clip embeddings on the GPU: the streamed head_dim-88 attention (cb_attention_stream_f16), the GEMM's erf-GELU and
LayerScale epilogues (cb_gemm_f16_ex), the RMSNorms, the tower (cb_iv2_*) against the reference's own module (golden vectors) and
against oracle/internvideo2.py at full depth, and InternVideo2FrameCreationStage -> InternVideo2EmbeddingStage."""

from __future__ import annotations

import json
import os
import uuid

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden
from gpu_helpers import ctx  # noqa: F401
from oracle import attention as A
from oracle import internvideo2 as O

pytestmark = pytest.mark.gpu

HD = 88
PAD = 3
SENTINEL = -7777.0
KINDS = ("normal", "sharp", "large", "ties")
SWEEP_T = [1, 2, 63, 64, 65, 127, 128, 129, 1024, 1025, 1026, 2049]


# ------------------------------------------------------------------------------------------------------------- attention
def _call(ctx, qkv_ptr, out_ptr, n, t, heads, hd) -> int:
    from cosmos_curate_b200.runtime import _stream_ptr

    return ctx.lib.cb_attention_stream_f16(ctx.h, qkv_ptr, out_ptr, n, t, heads, hd, _stream_ptr())


def _run(ctx, qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """cb_attention_stream_f16 on qkv placed between NaN rows, writing into a sentinel-filled buffer; asserts nothing outside the
    output was written."""
    from cosmos_curate_b200.runtime import check

    n, t, three_hidden = qkv.shape
    hidden, rows = three_hidden // 3, n * t
    src = torch.full((rows + 2 * PAD, three_hidden), float("nan"), dtype=torch.float16, device="cuda")
    src[PAD : PAD + rows] = qkv.reshape(rows, three_hidden)
    dst = torch.full((rows + 2 * PAD, hidden), SENTINEL, dtype=torch.float16, device="cuda")
    check(_call(ctx, src[PAD:].data_ptr(), dst[PAD:].data_ptr(), n, t, heads, HD), "cb_attention_stream_f16", ctx.h)
    torch.cuda.synchronize()
    assert (dst[:PAD] == SENTINEL).all() and (dst[PAD + rows :] == SENTINEL).all(), "rows outside [n*T][hidden] were written"
    return dst[PAD : PAD + rows].view(n, t, hidden)


def _assert_bitwise(got, want, what):
    bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
    if len(bad):
        i, tok, col = bad[0].tolist()
        pytest.fail(f"{what}: {len(bad)} elements differ; first at clip {i} token {tok} column {col}: got {got[i, tok, col].item()} want {want[i, tok, col].item()}")


@pytest.fixture(scope="module")
def worst():
    w = {"ratio": 0.0}
    yield w
    print(f"\nattention_stream: worst err/bound {w['ratio']:.3f}")


@pytest.mark.parametrize("t", SWEEP_T)
def test_attention_stream_sweep(ctx, worst, t):
    n, heads = (2, 2) if t < 1000 else (1, 3)
    seed = t * 100 + HD
    if t <= 2 ** A.SELECT_BITS:  # the selection code has 11 bits: T <= 2048
        qkv, pi = A.selection_inputs(n, t, heads, HD, seed)
        want = A.merge_heads(torch.gather(A.split_heads(qkv, heads)[2], 2, pi[..., None].expand(-1, -1, -1, HD)))
        _assert_bitwise(_run(ctx, qkv.cuda(), heads), want.cuda(), "selection")
    qkv, c = A.uniform_inputs(n, t, heads, HD, seed)
    _assert_bitwise(_run(ctx, qkv.cuda(), heads), A.merge_heads(c[:, :, None, :].expand(n, heads, t, HD)).half().cuda(), "uniform")
    for kind in KINDS:
        qkv = A.random_inputs(n, t, heads, HD, seed, kind=kind).cuda()
        got = _run(ctx, qkv, heads).double()
        ref, s_abs = A.reference(qkv, heads)
        ratio = ((got - ref).abs() / A.bound(ref, s_abs, qkv, heads)).max().item()
        worst["ratio"] = max(worst["ratio"], ratio)
        assert ratio <= 1.0, f"{kind}: err/bound {ratio:.3f}"


@pytest.mark.parametrize("t", [65, 1025])
def test_attention_stream_poisoned_neighbour_clip_and_head(ctx, t):
    """Clip 1 of 3 is Inf/NaN everywhere; in clips 0 and 2, head 1's Q, K and V columns are NaN.  Heads 0 and 2 of clips 0 and 2 stay
    finite and equal, bit for bit, to runs where the poisoned columns hold finite values."""
    heads = 3
    clean = A.random_inputs(3, t, heads, HD, seed=t).cuda()
    qkv = clean.clone()
    pattern = torch.tensor([float("inf"), float("nan"), float("-inf")], dtype=torch.float16, device="cuda")
    qkv[1] = pattern[torch.arange(qkv.shape[2], device="cuda") % 3]
    hidden = heads * HD
    for part in range(3):
        qkv[[0, 2], :, part * hidden + HD : part * hidden + 2 * HD] = float("nan")
    out = _run(ctx, qkv, heads)
    ref = _run(ctx, clean, heads)
    keep = torch.cat([torch.arange(0, HD), torch.arange(2 * HD, 3 * HD)]).cuda()
    for b in (0, 2):
        assert torch.isfinite(out[b][:, keep]).all(), f"clip {b}: a poisoned neighbour reached heads 0 / 2"
        _assert_bitwise(out[b : b + 1][:, :, keep], ref[b : b + 1][:, :, keep], f"clip {b} next to poison vs clean")


def test_attention_stream_repeat_launches_bitwise_equal(ctx):
    qkv = A.random_inputs(3, 1025, 4, HD, seed=5, kind="sharp").cuda()
    first = _run(ctx, qkv, 4)
    for _ in range(3):
        assert torch.equal(first, _run(ctx, qkv, 4))


def test_attention_stream_many_units(ctx):
    """More (clip, head, 128-row block) units than SMs, one clip per 16 heads as in the tower: every unit against the reference."""
    qkv = A.random_inputs(8, 1025, 16, HD, seed=8).cuda()
    got = _run(ctx, qkv, 16).double()
    ref, s_abs = A.reference(qkv, 16)
    assert ((got - ref).abs() / A.bound(ref, s_abs, qkv, 16)).max().item() <= 1.0


@pytest.mark.parametrize("hd", [64, 72, 80, 96])
def test_attention_stream_other_head_dims_unsupported(ctx, hd):
    t, heads = 100, 2
    qkv = torch.zeros(t, 3 * heads * hd, dtype=torch.float16, device="cuda")
    out = torch.full((t, heads * hd), SENTINEL, dtype=torch.float16, device="cuda")
    assert _call(ctx, qkv.data_ptr(), out.data_ptr(), 1, t, heads, hd) == -3  # CB_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()


def test_attention_stream_zero_clips_is_a_no_op(ctx):
    qkv = torch.full((1025, 3 * 2 * HD), float("nan"), dtype=torch.float16, device="cuda")
    out = torch.full((1025, 2 * HD), SENTINEL, dtype=torch.float16, device="cuda")
    assert _call(ctx, qkv.data_ptr(), out.data_ptr(), 0, 1025, 2, HD) == 0
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()


# ------------------------------------------------------------------------------------------------------------------- GEMM
def _operands(m, n, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(m, k, generator=g, device="cuda").half()
    w = (torch.randn(n, k, generator=g, device="cuda") / k**0.5).half()
    bias = torch.randn(n, generator=g, device="cuda") * 0.1
    return a, w, bias


@pytest.mark.parametrize(("m", "n", "k"), [(1025, 6144, 1408), (300, 4224, 1408), (77, 768, 1408), (8, 512, 768)])
def test_gemm_gelu_erf(ctx, m, n, k):
    from cosmos_curate_b200 import _lib

    a, w, bias = _operands(m, n, k, seed=m + n)
    got = ctx.gemm(a, w, bias=bias, epilogue=_lib.EPI_GELU_ERF).double()
    pre = a.double() @ w.double().T + bias.double()
    ref = torch.nn.functional.gelu(pre)
    acc_err = k * 2.0**-23 * (a.double().abs() @ w.double().abs().T)  # fp32 accumulation; |gelu'| <= 1.13
    assert ((got - ref).abs() <= 2.0**-11 * ref.abs() + 1.13 * acc_err + 2.0**-22 * pre.abs() + 2.0**-24).all()


@pytest.mark.parametrize(("m", "n", "k", "gamma_kind"), [(1025, 1408, 1408, "uniform"), (300, 1408, 6144, "uniform"), (77, 768, 1408, "uniform"),
                                                        (1025, 1408, 1408, "init"), (130, 4224, 1408, "uniform")])  # fmt: skip
def test_gemm_layerscale_residual_in_place(ctx, m, n, k, gamma_kind):
    """out = residual + gamma * (A W^T + bias), residual aliased with the output, inside a sentinel-filled buffer."""
    a, w, bias = _operands(m, n, k, seed=3 * m + n)
    gamma = torch.rand(n, device="cuda") * 1.45 + 0.05 if gamma_kind == "uniform" else torch.full((n,), 1e-5, device="cuda")
    res0 = torch.randn(m, n, device="cuda")
    buf = torch.full((m + 2 * PAD, n), SENTINEL, device="cuda")
    buf[PAD : PAD + m] = res0
    res = buf[PAD : PAD + m]
    out = ctx.gemm_ex(a, w, bias=bias, gamma=gamma, residual=res, out_f32=True)
    torch.cuda.synchronize()
    assert out.data_ptr() == res.data_ptr()
    assert (buf[:PAD] == SENTINEL).all() and (buf[PAD + m :] == SENTINEL).all()
    upd = gamma.double() * (a.double() @ w.double().T + bias.double())
    ref = res0.double() + upd
    tol = gamma.double() * k * 2.0**-23 * (a.double().abs() @ w.double().abs().T) + 2.0**-23 * (ref.abs() + upd.abs()) + 1e-30
    assert ((out.double() - ref).abs() <= tol).all()
    # without a residual, the scaled update alone: at gamma = 1e-5 it keeps its relative precision (gamma is not folded into fp16 weights)
    alone = ctx.gemm_ex(a, w, bias=bias, gamma=gamma, out_f32=True).double()
    assert ((alone - upd).abs() <= tol).all()


def test_gemm_layerscale_rows_do_not_depend_on_their_place(ctx):
    """Rows 1025.. of a 2050-row product equal, bit for bit, the same rows computed alone (they sit in other slots of the tiles)."""
    a, w, bias = _operands(2050, 1408, 1408, seed=4)
    gamma = torch.rand(1408, device="cuda") + 0.1
    res = torch.randn(2050, 1408, device="cuda")
    whole = ctx.gemm_ex(a, w, bias=bias, gamma=gamma, residual=res.clone(), out_f32=True)
    part = ctx.gemm_ex(a[1025:].contiguous(), w, bias=bias, gamma=gamma, residual=res[1025:].clone(), out_f32=True)
    assert torch.equal(whole[1025:], part)


def test_gemm_ex_without_gamma_is_cb_gemm_f16(ctx):
    a, w, bias = _operands(1025, 1408, 1408, seed=1)
    res = torch.randn(1025, 1408, device="cuda")
    r1, r2 = res.clone(), res.clone()
    assert torch.equal(ctx.gemm(a, w, bias=bias, residual=r1, out_f32=True), ctx.gemm_ex(a, w, bias=bias, residual=r2, out_f32=True))


# ------------------------------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize(("rows", "d"), [(1025, 1408), (37, 1408), (5, 768)])
def test_rmsnorm(ctx, rows, d):
    x = torch.randn(rows, d, device="cuda") * 3 + 0.5
    w = 1 + 0.2 * torch.randn(d, device="cuda")
    got = ctx.rmsnorm(x, w, 1e-6).double()
    xd = x.double()
    ref = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6)
    assert ((got - ref).abs() <= 2.0**-11 * ref.abs() + 1e-5 * ref.abs() + 2.0**-24).all()


@pytest.mark.parametrize(("rows", "d"), [(1025, 1408), (9, 1408), (3, 256)])
def test_qk_rmsnorm_in_place(ctx, rows, d):
    qkv = (torch.randn(rows, 3 * d, device="cuda") * 2).half()
    wq, wk = 1 + 0.2 * torch.randn(d, device="cuda"), 1 + 0.2 * torch.randn(d, device="cuda")
    before = qkv.clone()
    ctx.qk_rmsnorm_(qkv, wq, wk, 1e-6)
    torch.cuda.synchronize()
    assert torch.equal(qkv[:, 2 * d :], before[:, 2 * d :])  # V untouched
    for part, w in ((0, wq), (1, wk)):
        xd = before[:, part * d : (part + 1) * d].double()
        ref = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6)
        got = qkv[:, part * d : (part + 1) * d].double()
        assert ((got - ref).abs() <= 2.0**-11 * ref.abs() + 1e-5 * ref.abs() + 2.0**-24).all(), part


# ------------------------------------------------------------------------------------------------------------------- tower
def _errors(got: np.ndarray, want: np.ndarray):
    cos = (got * want).sum(-1) / (np.linalg.norm(got, axis=-1) * np.linalg.norm(want, axis=-1))
    return float(1 - cos.min()), float(np.abs(got - want).max())


def test_tower_matches_the_reference_module(ctx):
    """cb_iv2_forward on the golden cases (the reference's PretrainInternVideo2 in float32 at depth 2, 1408 wide): cosine >= 1 - 1e-5,
    max-abs <= 1e-3 on the unit-norm embeddings; the reference's own bf16 run on the same inputs is printed beside it."""
    from cosmos_curate_b200.runtime import Iv2Tower

    g = load_golden("internvideo2_ref.npz")
    meta = json.loads(bytes(g["meta"]).decode())
    for case in meta["cases"]:
        cfg = O.IV2_1B.with_(frames=case["frames"], layers=meta["depth"])
        gamma = tuple(case["gamma"]) if isinstance(case["gamma"], list) else case["gamma"]
        w = O.random_weights(cfg, case["seed"], gamma)
        tubes = torch.from_numpy(O.tube_from_frames(O.expand_frames(g["frames_u8"][:, : case["frames"]], meta["block"]))).cuda()
        tower = Iv2Tower(ctx, cfg.to_dict(), w, max_clips=2)
        got = tower.forward(tubes).cpu().numpy()
        one = np.concatenate([tower.forward(tubes[i : i + 1]).cpu().numpy() for i in range(2)])
        tower.close()
        want = g[f"{case['name']}_emb"]
        e_cos, e_abs = _errors(got, want)
        b_cos, b_abs = _errors(g[f"{case['name']}_emb_bf16"], want)
        print(f"\n{case['name']}: tower 1-cos {e_cos:.2e} max-abs {e_abs:.2e} | reference bf16 1-cos {b_cos:.2e} max-abs {b_abs:.2e} | "
              f"batch-of-1 max diff {np.abs(one - got).max():.1e}")  # fmt: skip
        assert e_cos <= 1e-5 and e_abs <= 1e-3, case["name"]
        assert np.array_equal(one, got)  # a clip's embedding does not depend on its batch neighbour or its rows' place in the batch


def test_tower_full_depth_against_the_oracle(ctx):
    """40 layers at 1408 wide, 4 frames, seeded weights with LayerScale gammas ~ U(0.1, 1): fp16 GEMM operands vs the float32 oracle."""
    from cosmos_curate_b200.runtime import Iv2Tower

    cfg = O.IV2_1B
    w = O.random_weights(cfg, seed=21, gamma=(0.1, 1.0))
    frames = np.random.default_rng(22).integers(0, 256, (3, 4, 224, 224, 3), dtype=np.uint8)
    tubes = torch.from_numpy(O.tube_from_frames(frames)).cuda()
    tower = Iv2Tower(ctx, cfg.to_dict(), w, max_clips=2)  # 3 clips: two chunks
    got = tower.forward(tubes).cpu().numpy()
    tower.close()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            want = O.forward(cfg, w, tubes, device="cuda").cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    for i in range(3):
        e_cos, e_abs = _errors(got[i : i + 1], want[i : i + 1])
        print(f"\nfull depth clip {i}: 1-cos {e_cos:.2e} max-abs {e_abs:.2e}")
    e_cos, e_abs = _errors(got, want)
    assert e_cos <= 1e-5 and e_abs <= 1e-3


def test_frame_creation_then_embedding_stage(ctx):
    """InternVideo2FrameCreationStage(num_frames=4) -> InternVideo2EmbeddingStage on coded clips, a broken clip and a too-short clip:
    the embeddings equal cb_iv2_forward on the tubes the first stage made."""
    from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
    from cosmos_curate_b200.models.internvideo2 import IV2_1B_CFG, InternVideo2MultiModality
    from cosmos_curate_b200.models.internvideo2_frames import InternVideo2FrameFormulator
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage, InternVideo2FrameCreationStage
    from tools import synth_h264

    sintel = (GOLDEN / "sintel_clip_10s.mp4").read_bytes()
    synth = synth_h264.make_clip(640, 360, 30, 3.0, seed=5, gop=30, pan=(2, 1))
    tiny = synth_h264.make_clip(320, 192, 30, 0.1, seed=3, gop=30)  # 3 frames: too short at any rate up to 20 fps
    datas = [sintel, synth, b"\x00" * 4096, tiny, None]
    clips = [Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, 3.0), encoded_data=d) for d in datas]
    tasks = [SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips[:3])),
             SplitPipeTask(session_id="s", video=Video(input_video="w.mp4", clips=clips[3:]))]  # fmt: skip
    frames_stage = InternVideo2FrameCreationStage(target_fps=2.0, source="nvdec", model=InternVideo2FrameFormulator(num_frames=4))
    frames_stage.stage_setup()
    frames_stage.process_data(tasks)
    tubes = [c.intern_video_2_frames.resolve() for c in clips]
    assert tubes[0].shape == (1, 4, 3, 224, 224) and tubes[1].shape == (1, 4, 3, 224, 224) and tubes[3].shape == (0,)
    assert clips[2].errors["frame_extraction"] == "video_decode_failed"
    tubes = [None if t is None else t.copy() for t in tubes]

    model = InternVideo2MultiModality(seed=7, config=dict(IV2_1B_CFG, layers=2), max_clips=8)
    stage = InternVideo2EmbeddingStage(batch_size=8, log_stats=True, model=model)
    stage.stage_setup()
    assert model.get_target_num_frames() == 4
    stage.process_data(tasks)
    assert clips[3].errors == {"iv2_frames": "empty"} and clips[4].errors == {"encoded_data": "empty", "iv2_frames": "none"}
    assert clips[2].errors.get("iv2_frames") == "none" and clips[2].intern_video_2_embedding is None
    assert all(c.intern_video_2_frames.resolve() is None for c in clips)
    direct = model.tower.forward(torch.from_numpy(np.concatenate([tubes[0], tubes[1]])).cuda()).cpu().numpy()
    for i in (0, 1):
        e = clips[i].intern_video_2_embedding
        assert e.shape == (1, 512) and e.dtype == np.float32
        np.testing.assert_array_equal(e[0], direct[i])
    # a tube of another frame count is refused, naming both counts
    bad = Clip(uuid=uuid.uuid4(), source_video="v.mp4", span=(0.0, 1.0))
    bad.intern_video_2_frames = np.zeros((1, 8, 3, 224, 224), np.float32)
    with pytest.raises(ValueError, match="8 frames, the InternVideo2 tower takes 4"):
        stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=[bad]))])


@pytest.mark.skipif(not os.environ.get("CURATE_B200_IV2_CHECKPOINT"), reason="set CURATE_B200_IV2_CHECKPOINT to InternVideo2-stage2_1b-224p-f4.pt")
def test_reference_real_weight_checkpoint(ctx):
    """The real checkpoint through the model class vs oracle/internvideo2.py in float32 on the same weights."""
    from cosmos_curate_b200.models.internvideo2 import InternVideo2MultiModality

    model = InternVideo2MultiModality(checkpoint=os.environ["CURATE_B200_IV2_CHECKPOINT"])
    model.setup()
    assert model.get_target_num_frames() == 4
    frames = np.random.default_rng(3).integers(0, 256, (2, 4, 224, 224, 3), dtype=np.uint8)
    tubes = O.tube_from_frames(frames)
    got = np.concatenate(model.encode_batched_videos([t[None] for t in tubes], 8))
    with torch.no_grad():
        want = O.forward(O.IV2_1B, model._load_weights(), torch.from_numpy(tubes), device="cuda").cpu().numpy()
    e_cos, e_abs = _errors(got, want)
    print(f"\nreal checkpoint: 1-cos {e_cos:.2e} max-abs {e_abs:.2e}")
    assert e_cos <= 1e-5 and e_abs <= 1e-3
