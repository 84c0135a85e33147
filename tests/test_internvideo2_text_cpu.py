"""InternVideo2 text tower, host side: the tokenizer against the reference tokenizer's ids (tests/golden/internvideo2_text_tokens.json),
the [CLS] / [SEP] / [PAD] assembly, the torch restatement (oracle/internvideo2_text.py) against the reference's own BertModel
(tests/golden/internvideo2_text_ref.npz), the checkpoint key mapping, `evaluate`, and InternVideo2EmbeddingStage's texts_to_verify
contract with a fake model."""

from __future__ import annotations

import json
import uuid

import numpy as np
import pytest
import torch

from conftest import GOLDEN, golden_json, load_golden
from cosmos_curate_b200.data_model import Clip, SplitPipeTask, Video
from cosmos_curate_b200.models import internvideo2 as M
from cosmos_curate_b200.models.bert_tokenizer import BertTokenizer
from oracle import internvideo2_text as O


def _tokens_golden():
    return json.loads((GOLDEN / "internvideo2_text_tokens.json").read_text(encoding="utf-8"))


def _tokenizer() -> BertTokenizer:
    return BertTokenizer.from_file(GOLDEN / _tokens_golden()["vocab"])


def test_tokenizer_matches_the_reference_tokenizer():
    g = _tokens_golden()
    tok = _tokenizer()
    assert len(g["cases"]) >= 20
    for case in g["cases"]:
        assert tok.tokenize(case["text"]) == case["tokens"], repr(case["text"])
        assert tok.ids(case["text"]) == case["ids"], repr(case["text"])


def test_assembly_cls_sep_truncation_padding():
    tok = _tokenizer()
    v = tok.vocab
    texts = ["a dog", "", " ".join(["red"] * 38), " ".join(["red"] * 39), " ".join(["blue"] * 100), "\t\n"]
    ids, lengths = tok(texts, 40)
    assert ids.dtype == np.int32 and lengths.dtype == np.int32 and ids.shape == (6, 40)
    assert lengths.tolist() == [4, 2, 40, 40, 40, 2]
    for row, n, text in zip(ids, lengths, texts):
        pieces = tok.ids(text)[:38]
        assert row[0] == v["[CLS]"] and row[n - 1] == v["[SEP]"] and (row[n:] == v["[PAD]"]).all()
        assert row[1 : n - 1].tolist() == pieces
    assert ids[4, 1:39].tolist() == [v["blue"]] * 38  # truncated to 38 pieces, then [SEP]
    with pytest.raises(ValueError, match="no room"):
        tok(["a"], 1)


def test_tower_golden_ids_are_this_tokenizers():
    g = load_golden("internvideo2_text_ref.npz")
    meta = golden_json(g, "meta")
    ids, lengths = _tokenizer()(meta["texts"], 40)
    assert np.array_equal(ids, g["ids"]) and np.array_equal(lengths, g["lengths"])
    assert 40 in lengths.tolist() and lengths.min() < 10  # one text fills 40 tokens exactly (another is truncated), others are short


def test_oracle_matches_the_reference_bert_in_float32():
    g = load_golden("internvideo2_text_ref.npz")
    meta = golden_json(g, "meta")
    cfg = O.IV2_TEXT.with_(layers=meta["depth"], vocab=meta["vocab"])
    got = O.forward(cfg, O.random_weights(cfg, meta["seed"]), g["ids"], g["lengths"]).numpy()
    want = g["emb"]
    rel = np.linalg.norm(got - want, axis=1) / np.linalg.norm(want, axis=1)
    assert rel.max() <= 2e-5, rel
    # the reference's own bf16 run is much further away: the scale the GPU tower's 1e-3 bound is measured against
    assert np.abs(g["emb_bf16"] - want).max() > 1e-4


def test_oracle_ignores_padding():
    cfg = O.IV2_TEXT.with_(hidden=128, heads=2, mlp=256, vocab=50, max_pos=16, layers=2, embed_dim=32)
    w = O.random_weights(cfg, 3)
    ids = np.array([[1, 5, 7, 2, 0, 0, 0, 0]])
    a = O.forward(cfg, w, ids, [4])
    b = O.forward(cfg, w, ids[:, :4], [4])
    c = O.forward(cfg, w, np.where(np.arange(8) < 4, ids, 9), [4])  # other values in the padding
    assert torch.allclose(a, b, atol=1e-6) and torch.equal(a, c)


def test_flops_formula():
    assert abs(O.flops_per_text(O.IV2_TEXT) / 1e9 - 19.25) < 0.05


SMALL = {"hidden": 128, "layers": 2, "heads": 2, "mlp": 256, "vocab": 50, "max_pos": 16, "embed_dim": 32, "ln_eps": 1e-12}


def _reference_text_state_dict(cfg: dict, w: dict) -> dict:
    """`w` under the reference checkpoint's text keys and shapes (token_type_embeddings [2][d], split q/k/v), plus extra layers and
    vision keys the loader must ignore."""
    sd = {}
    for name, a in w.items():
        keys = M.text_reference_keys(name)
        t = torch.from_numpy(a.copy())
        if name == "type_emb":
            t = torch.stack([t, torch.full_like(t, 7.0)])
        for k, part in zip(keys, t.chunk(len(keys), 0)):
            sd[k] = part.clone()
    sd[f"text_encoder.bert.encoder.layer.{cfg['layers']}.attention.self.query.weight"] = torch.zeros(4, 4)
    sd["text_encoder.bert.encoder.layer.0.crossattention.self.query.weight"] = torch.zeros(4, 4)
    sd["vision_proj.weight"] = torch.zeros(4, 4)
    return sd


@pytest.mark.parametrize("wrap", ["model", "module"])
def test_text_checkpoint_round_trip(tmp_path, wrap):
    w = M.seeded_text_weights(SMALL, seed=4)
    assert w.keys() == M.text_tensor_shapes(SMALL).keys()
    keys = [k for n in w for k in M.text_reference_keys(n)]
    assert len(set(keys)) == len(keys) and all(k.startswith(("text_encoder.bert.", "text_proj.")) for k in keys)
    assert M.text_reference_keys("L3.qkv_b") == [f"text_encoder.bert.encoder.layer.3.attention.self.{x}.bias" for x in ("query", "key", "value")]
    path = tmp_path / "ckpt.pt"
    torch.save({wrap: _reference_text_state_dict(SMALL, w), "epoch": 1}, path)
    back = M.load_text_checkpoint(path, SMALL)
    assert back.keys() == w.keys()
    for name, a in w.items():
        assert back[name].dtype == np.float32 and np.array_equal(back[name], a), name


def test_text_checkpoint_missing_key_is_named(tmp_path):
    w = M.seeded_text_weights(SMALL, seed=4)
    sd = _reference_text_state_dict(SMALL, w)
    del sd["text_encoder.bert.encoder.layer.1.output.LayerNorm.bias"]
    path = tmp_path / "ckpt.pt"
    torch.save({"model": sd}, path)
    with pytest.raises(KeyError, match=r"text_encoder\.bert\.encoder\.layer\.1\.output\.LayerNorm\.bias"):
        M.load_text_checkpoint(path, SMALL)


def test_text_needs_a_vocab(monkeypatch, tmp_path):
    monkeypatch.delenv("CURATE_B200_WEIGHTS_DIR", raising=False)
    with pytest.raises(FileNotFoundError, match="vocab.txt"):
        M.InternVideo2MultiModality(seed=0).tokenizer  # noqa: B018
    small = dict(SMALL, vocab=10)
    with pytest.raises(ValueError, match="text tower embeds 10"):
        M.InternVideo2MultiModality(seed=0, text_config=small, vocab_file=GOLDEN / _tokens_golden()["vocab"]).tokenizer  # noqa: B018
    assert M.InternVideo2MultiModality(seed=0).encode_texts([]).shape == (0, 512)


# ---------------------------------------------------------------------------------------------------------------- evaluate
def test_evaluate_is_softmax_topk():
    rng = np.random.default_rng(0)
    for n in (1, 2, 7, 40):
        v = rng.standard_normal((1, 512)).astype(np.float32)
        v /= np.linalg.norm(v)
        t = [x[None] / np.linalg.norm(x) for x in rng.standard_normal((n, 512)).astype(np.float32)]
        probs, idxs = M.InternVideo2MultiModality.evaluate(torch.from_numpy(v), [torch.from_numpy(x) for x in t])
        want = (100.0 * torch.from_numpy(v) @ torch.from_numpy(np.concatenate(t)).T).softmax(dim=-1)
        wp, wi = want.topk(n, dim=-1)
        assert idxs == wi[0].tolist() and np.allclose(probs, wp[0].numpy(), rtol=0, atol=0)
        assert isinstance(probs[0], float) and isinstance(idxs[0], int)


def test_evaluate_ties_go_to_the_lower_index():
    v = np.zeros((1, 4), np.float32)
    v[0, 0] = 1
    t = [np.array([[0, 1, 0, 0]], np.float32), np.array([[1, 0, 0, 0]], np.float32), np.array([[0, 0, 1, 0]], np.float32),
         np.array([[1, 0, 0, 0]], np.float32)]  # fmt: skip
    probs, idxs = M.InternVideo2MultiModality.evaluate(v, t)
    assert idxs == [1, 3, 0, 2] and probs[0] == probs[1] and probs[2] == probs[3]


# --------------------------------------------------------------------------------------------------------- stage contract
class FakeTextModel:
    """Clip embeddings from the tube, text embeddings from the text: both fixed functions of their own input."""

    def __init__(self):
        self.text_calls: list[list[str]] = []

    def setup(self):
        pass

    @staticmethod
    def _unit(seed_bytes: bytes) -> np.ndarray:
        e = np.random.default_rng(list(seed_bytes) or [0]).standard_normal(512)
        return (e / np.linalg.norm(e)).astype(np.float32)

    def encode_batched_videos(self, videos, batch_size):
        return [self._unit(np.asarray(v, np.float32).tobytes()[:64])[None] for v in videos]

    def encode_texts(self, texts):
        self.text_calls.append(list(texts))
        return np.stack([self._unit(t.encode()) for t in texts])

    evaluate = staticmethod(M.InternVideo2MultiModality.evaluate)


def _clip(i, tube):
    c = Clip(uuid=uuid.uuid5(uuid.NAMESPACE_URL, f"iv2t_{i}"), source_video="v.mp4", span=(float(i), float(i + 1)))
    c.intern_video_2_frames = tube
    return c


def _tube(seed):
    return np.random.default_rng(seed).standard_normal((1, 4, 3, 8, 8)).astype(np.float32)


def test_stage_sets_the_text_match_where_the_embedding_exists():
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage

    texts = ["a dog", "a cat", "a car"]
    model = FakeTextModel()
    stage = InternVideo2EmbeddingStage(model=model, texts_to_verify=texts, batch_size=2)
    stage.stage_setup()
    clips = [_clip(0, _tube(0)), _clip(1, None), _clip(2, np.empty(0, np.float32)), _clip(3, _tube(3))]
    done = _clip(4, None)
    done.intern_video_2_embedding = model._unit(b"earlier")[None]  # embedded by an earlier run: matched too, as the reference does
    tasks = [SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips[:2])),
             SplitPipeTask(session_id="s", video=Video(input_video="w.mp4", clips=[*clips[2:], done]))]  # fmt: skip
    stage.process_data(tasks)
    stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="x.mp4", clips=[_clip(5, _tube(5))]))])
    t = model.encode_texts(texts)
    model.text_calls.pop()
    assert model.text_calls == [texts]  # once per stage, not once per clip
    assert clips[1].intern_video_2_text_match is None and clips[2].intern_video_2_text_match is None
    assert clips[1].errors == {"iv2_frames": "none"} and clips[2].errors == {"iv2_frames": "empty"}
    for c in (clips[0], clips[3], done):
        text, p = c.intern_video_2_text_match
        logits = 100.0 * (t @ c.intern_video_2_embedding.reshape(-1))
        probs = torch.from_numpy(logits.astype(np.float32)).softmax(-1).numpy()
        assert text == texts[int(np.argmax(probs))] and isinstance(p, float) and abs(p - probs.max()) < 1e-6


def test_stage_embeds_texts_at_first_use_without_setup():
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage

    model = FakeTextModel()
    stage = InternVideo2EmbeddingStage(model=model, texts_to_verify=["one", "two"])
    clips = [_clip(i, _tube(i)) for i in range(3)]
    stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=clips))])
    assert model.text_calls == [["one", "two"]] and all(c.intern_video_2_text_match[0] in ("one", "two") for c in clips)
    assert all(not c.errors for c in clips)


def test_stage_text_refusals():
    from cosmos_curate_b200.stages import InternVideo2EmbeddingStage

    with pytest.raises(ValueError, match="texts_to_verify"):
        InternVideo2EmbeddingStage(model=FakeTextModel(), texts_to_verify=[])

    class NoText:
        def encode_batched_videos(self, videos, batch_size):
            return []

    with pytest.raises(ValueError, match="texts_to_verify"):
        InternVideo2EmbeddingStage(model=NoText(), texts_to_verify=["a cat"])
    stage = InternVideo2EmbeddingStage(model=FakeTextModel())  # no texts: no match is set
    clip = _clip(0, _tube(0))
    stage.process_data([SplitPipeTask(session_id="s", video=Video(input_video="v.mp4", clips=[clip]))])
    assert clip.intern_video_2_embedding is not None and clip.intern_video_2_text_match is None
