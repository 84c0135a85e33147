"""InternVideo2 clip embeddings, host side: the torch restatement (oracle/internvideo2.py) against the reference's own module
(tests/golden/internvideo2_ref.npz), the checkpoint key mapping, InternVideo2EmbeddingStage's contract with a fake tower, the writer's
internvideo2 outputs, and the attention oracle at head_dim 88 (the streamed kernel's only head size)."""

from __future__ import annotations

import json
import uuid

import numpy as np
import pytest
import torch

from conftest import load_golden
from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
from cosmos_curate_b200.models import internvideo2 as M
from oracle import attention as A
from oracle import internvideo2 as O


def _golden():
    g = load_golden("internvideo2_ref.npz")
    return g, json.loads(bytes(g["meta"]).decode())


def _case_inputs(g, meta, case):
    cfg = O.IV2_1B.with_(frames=case["frames"], layers=meta["depth"])
    gamma = tuple(case["gamma"]) if isinstance(case["gamma"], list) else case["gamma"]
    return cfg, O.random_weights(cfg, case["seed"], gamma), O.tube_from_frames(O.expand_frames(g["frames_u8"][:, : case["frames"]], meta["block"]))


def test_oracle_matches_the_reference_module_in_float32():
    g, meta = _golden()
    assert {c["name"] for c in meta["cases"]} == {"t4", "t8", "t4_init_gamma"}
    for case in meta["cases"]:
        cfg, w, tubes = _case_inputs(g, meta, case)
        got = O.forward(cfg, w, tubes).numpy()
        want = g[f"{case['name']}_emb"]
        rel = np.linalg.norm(got - want, axis=1) / np.linalg.norm(want, axis=1)
        assert rel.max() <= 2e-5, (case["name"], rel)
        # the reference's own bf16 run is much further away: the gap the GPU tower's 1e-3 bound is measured against
        assert np.abs(g[f"{case['name']}_emb_bf16"] - want).max() > 1e-4


def test_flops_formula():
    assert abs(O.flops_per_clip(O.IV2_1B) / 1e12 - 2.3057) < 1e-3
    assert O.IV2_1B.tokens == 1025 and O.IV2_1B.with_(frames=8).tokens == 2049


def _reference_state_dict(cfg: dict, w: dict) -> dict:
    """`w` in the reference checkpoint's key layout and shapes, plus text-tower keys the loader must ignore."""
    sd = {}
    for name, a in w.items():
        t = torch.from_numpy(a.copy())
        if name == "patch_w":
            t = t.reshape(cfg["hidden"], 3, 1, cfg["patch"], cfg["patch"])
        elif name == "cls":
            t = t.reshape(1, 1, -1)
        elif name == "pos":
            t = t.reshape(1, -1, cfg["hidden"])
        sd[M.reference_key(name)] = t
    sd["text_encoder.bert.embeddings.word_embeddings.weight"] = torch.zeros(4, 8)
    sd["text_proj.weight"] = torch.zeros(512, 8)
    sd["vision_encoder.clip_decoder.0.head.weight"] = torch.zeros(8, 8)
    return sd


@pytest.mark.parametrize("wrap", ["model", "module"])
def test_checkpoint_round_trip(tmp_path, wrap):
    cfg = dict(M.IV2_1B_CFG, layers=2)
    w = M.seeded_weights(cfg, seed=5)
    keys = [M.reference_key(n) for n in w]
    assert len(set(keys)) == len(keys) and all(k.startswith(("vision_encoder.", "vision_proj.")) for k in keys)
    path = tmp_path / "ckpt.pt"
    torch.save({wrap: _reference_state_dict(cfg, w), "epoch": 3}, path)
    back = M.load_checkpoint(path, cfg)
    assert back.keys() == w.keys()
    for name, a in w.items():
        assert back[name].dtype == np.float32 and np.array_equal(back[name], a), name
    model = M.InternVideo2MultiModality(checkpoint=path, config=cfg)
    assert model.get_target_num_frames() == 4 and model.model_id_names == ["OpenGVLab/InternVideo2-Stage2_1B-224p-f4"]


def test_checkpoint_with_another_frame_count_is_refused(tmp_path):
    cfg = dict(M.IV2_1B_CFG, layers=1)
    w = M.seeded_weights(dict(cfg, frames=8), seed=1)
    path = tmp_path / "f8.pt"
    torch.save({"model": _reference_state_dict(cfg, w)}, path)
    with pytest.raises(ValueError, match="8 frames, the tower takes 4"):
        M.load_checkpoint(path, cfg)


def test_missing_weights_are_an_error(monkeypatch):
    monkeypatch.delenv("CURATE_B200_SYNTHETIC_WEIGHTS", raising=False)
    monkeypatch.delenv("CURATE_B200_WEIGHTS_DIR", raising=False)
    with pytest.raises(FileNotFoundError, match="synthetic weights were not requested"):
        M.InternVideo2MultiModality().get_target_num_frames()
    assert M.InternVideo2MultiModality(seed=0, config=dict(M.IV2_1B_CFG, layers=1)).get_target_num_frames() == 4


# ---------------------------------------------------------------------------------------------------------- stage contract
class FakeTower:
    """Stands in for the GPU tower: each clip's embedding is a fixed function of its own tube."""

    frames = 4

    def __init__(self):
        self.calls: list[int] = []

    def encode_batched_videos(self, videos, batch_size):
        out = []
        for i in range(0, len(videos), batch_size):
            chunk = videos[i : i + batch_size]
            self.calls.append(len(chunk))
            for v in chunk:
                a = np.asarray(v, dtype=np.float32)[0]
                if a.shape[0] != self.frames:
                    msg = f"tube has {a.shape[0]} frames, the InternVideo2 tower takes {self.frames}"
                    raise ValueError(msg)
                e = np.resize(a.reshape(-1)[:4096].astype(np.float64), 512) + np.arange(512)
                out.append((e / np.linalg.norm(e)).astype(np.float32)[None])
        return out

    def setup(self):
        pass


def _clip(i, tube):
    c = Clip(uuid=uuid.uuid5(uuid.NAMESPACE_URL, f"iv2_{i}"), source_video="v.mp4", span=(float(i), float(i + 1)))
    c.intern_video_2_frames = tube
    return c


def _tube(seed, frames=4, size=8):
    return np.random.default_rng(seed).standard_normal((1, frames, 3, size, size)).astype(np.float32)


def _stage(**kw):
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage

    tower = FakeTower()
    return InternVideo2EmbeddingStage(model=tower, **kw), tower


def test_stage_contract_with_a_fake_tower():
    stage, tower = _stage(batch_size=2, log_stats=True)
    assert stage.resources.gpus == 0.25
    clips = [_clip(0, _tube(0)), _clip(1, None), _clip(2, np.empty(0, dtype=np.float32)), _clip(3, _tube(3)), _clip(4, _tube(4))]
    tasks = [SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips[:3])),
             SplitPipeTask(session_id="s", video=Video(input_video="w.mp4", clips=clips[3:]))]  # fmt: skip
    assert stage.process_data(tasks) == tasks
    assert clips[1].errors == {"iv2_frames": "none"} and clips[2].errors == {"iv2_frames": "empty"}
    assert clips[1].intern_video_2_embedding is None and clips[2].intern_video_2_embedding is None
    for c in (clips[0], clips[3], clips[4]):
        e = c.intern_video_2_embedding
        assert e.shape == (1, 512) and e.dtype == np.float32 and abs(np.linalg.norm(e) - 1) < 1e-5 and not c.errors
    assert all(c.intern_video_2_frames.resolve() is None for c in clips)  # dropped for every clip
    assert tower.calls == [2, 1]  # clips of both tasks share the batches
    assert "InternVideo2EmbeddingStage" in tasks[0].stage_perf and "InternVideo2EmbeddingStage" in tasks[1].stage_perf


def test_stage_output_does_not_depend_on_batch_composition():
    tubes = [_tube(10 + i) for i in range(5)]
    results = []
    for bs, order in ((8, [0, 1, 2, 3, 4]), (1, [0, 1, 2, 3, 4]), (2, [4, 2, 0, 3, 1])):
        stage, _ = _stage(batch_size=bs)
        clips = [_clip(i, tubes[i]) for i in order]
        stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips))])
        results.append({c.uuid: c.intern_video_2_embedding for c in clips})
    for r in results[1:]:
        assert all(np.array_equal(r[k], results[0][k]) for k in results[0])


def test_stage_refusals():
    with pytest.raises(ValueError, match="texts_to_verify"):
        _stage(texts_to_verify=["a cat"])
    stage, _ = _stage()
    clip = _clip(0, _tube(0, frames=8))
    with pytest.raises(ValueError, match="8 frames, the InternVideo2 tower takes 4"):
        stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=[clip]))])
    assert clip.intern_video_2_frames.resolve() is None


def test_real_model_refuses_a_tube_of_another_frame_count():
    model = M.InternVideo2MultiModality(seed=0, config=dict(M.IV2_1B_CFG, layers=1))

    class _T:
        frames = 4

    model._tower = _T()
    with pytest.raises(ValueError, match="tube has 8 frames, the InternVideo2 tower takes 4"):
        model.encode_batched_videos([np.zeros((1, 8, 3, 224, 224), np.float32)], 8)


def test_writer_internvideo2_embeddings_read_back(tmp_path):
    from cosmos_curate_b200 import embedding_io as E
    from cosmos_curate_b200.stages import ClipWriterStage

    stage, _ = _stage()
    clips = [_clip(i, _tube(20 + i)) for i in range(3)]
    v = Video(input_video="/data/in/a.mp4", relative_path="a", clips=clips, clip_chunk_index=0)
    task = SplitPipeTask(session_id="s", video=v)
    stage.process_data([task])
    want = {str(c.uuid): c.intern_video_2_embedding.copy() for c in clips}
    writer = ClipWriterStage(str(tmp_path), "/data/in/", upload_clips=False, upload_clip_info_in_chunks=False, generate_embeddings=True,
                             embedding_algorithm="internvideo2")  # fmt: skip
    writer.process_data([task])
    ids, x = E.read_embedding_parquets(sorted((tmp_path / "iv2_embd_parquet").glob("*.parquet")))
    assert x.shape == (3, 512) and x.dtype == np.float32
    assert all(np.array_equal(x[i], want[ids[i]].reshape(-1)) for i in range(3))


# -------------------------------------------------------------------------------------------- attention oracle at head_dim 88
HD = 88
SWEEP_T = [1, 2, 63, 64, 65, 127, 128, 129, 1024, 1025, 1026, 2049]


@pytest.mark.parametrize("t", [1, 65, 129, 1025])
def test_selection_is_one_hot_at_head_dim_88(t):
    qkv, pi = A.selection_inputs(2, t, 2, HD, seed=t)
    assert torch.equal(torch.from_numpy(A.emulate(qkv.numpy(), 2)), A.merge_heads(torch.gather(A.split_heads(qkv, 2)[2], 2, pi[..., None].expand(-1, -1, -1, HD))))


def test_uniform_gives_the_constant_exactly_at_head_dim_88():
    qkv, c = A.uniform_inputs(2, 1025, 2, HD, seed=1)
    assert torch.equal(torch.from_numpy(A.emulate(qkv.numpy(), 2)), A.merge_heads(c[:, :, None, :].expand(2, 2, 1025, HD)).half())


@pytest.mark.parametrize("kind", ["normal", "sharp", "large", "ties"])
def test_emulated_kernel_within_the_bound_at_head_dim_88(kind):
    worst = 0.0
    for i, t in enumerate([1, 2, 63, 65, 129, 1025]):
        qkv = A.random_inputs(1, t, 2, HD, seed=100 * i + 7, kind=kind)
        ref, s_abs = A.reference(qkv, 2)
        err = (torch.from_numpy(A.emulate(qkv.numpy(), 2)).double() - ref).abs()
        worst = max(worst, (err / A.bound(ref, s_abs, qkv, 2)).max().item())
    assert worst <= 0.7, worst
    assert A.path_of(1025, HD) is None  # cb_attention_f16 does not take head_dim 88; cb_attention_stream_f16 does
