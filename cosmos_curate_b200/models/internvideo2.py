"""InternVideo2 clip and text embeddings on the H100 path: the `ModelInterface` of the reference's InternVideo2MultiModality
(cosmos_curate/models/internvideo2_mm.py:306-512).
  * vision: `encode_batched_videos` returns one unit-norm float32 [1, 512] array per clip (InternVideo2_Stage2.get_vid_feat,
    :203-217, then np.split, :460-479);
  * text: `encode_texts` / `get_text_embedding` embed captions into the same 512-d space (get_txt_feat, :219-241: BERT-large's first
    19 layers, [CLS], text_proj, L2 norm) and `evaluate` ranks texts for a clip (predict_label, :243-254).  The text tower is a
    separate GPU handle, built at the first text call (or by setup_text()): a vision-only user never loads its weights.

Weights: the reference's checkpoint (InternVideo2-stage2_1b-224p-f4.pt, torch.load(weights_only=True), state dict under "model" or
"module"): vision_encoder.* and vision_proj.* for the vision tower, text_encoder.bert.embeddings.*, text_encoder.bert.encoder.layer.{0..18}.*
and text_proj.* for the text tower.  The vocabulary is google-bert/bert-large-uncased's vocab.txt (models/bert_tokenizer.py).  Seeded
synthetic weights only when explicitly requested (models/_weights_source.py); they still need a vocab.txt.
"""

from __future__ import annotations

import math
import os
from pathlib import Path

import numpy as np
import torch

from ..interfaces import ModelInterface
from ..runtime import Iv2TextTower, Iv2Tower, get_context
from . import _weights_source as src
from .bert_tokenizer import BERT_VOCAB_ID, BertTokenizer

_IV2_MODEL_ID = "OpenGVLab/InternVideo2-Stage2_1B-224p-f4"
CHECKPOINT_NAME = "InternVideo2-stage2_1b-224p-f4.pt"

# pretrain_internvideo2_1b_patch14_224 (internvideo2.py:696-735) with the shipped config (internvideo2_mm_config_model.json:390-461)
IV2_1B_CFG = {"image_size": 224, "patch": 14, "frames": 4, "hidden": 1408, "layers": 40, "heads": 16, "mlp": 6144, "clip_dim": 768,
              "embed_dim": 512, "rms_eps": 1e-6, "ln_eps": 1e-5}  # fmt: skip


# the text encoder of the same checkpoint: BERT-large (internvideo2_mm_config_bert.json) run in mode="text", i.e. its first
# fusion_layer = 19 layers (xbert.py:730-733), then text_proj 1024 -> 512; captions are tokenized to max_txt_l = 40 tokens
IV2_TEXT_CFG = {"hidden": 1024, "layers": 19, "heads": 16, "mlp": 4096, "vocab": 30522, "max_pos": 512, "embed_dim": 512, "ln_eps": 1e-12}
MAX_TXT_L = 40


def reference_key(name: str) -> str:
    """The reference checkpoint key of tower tensor `name` (cb_iv2_set_tensor's names)."""
    ve = "vision_encoder."
    fixed = {"patch_w": ve + "patch_embed.proj.weight", "patch_b": ve + "patch_embed.proj.bias", "cls": ve + "cls_token", "pos": ve + "pos_embed",
             "pool.proj_w": ve + "clip_projector.cross_attn.proj.weight", "pool.proj_b": ve + "clip_projector.cross_attn.proj.bias",
             "vproj_w": "vision_proj.weight", "vproj_b": "vision_proj.bias"}  # fmt: skip
    if name in fixed:
        return fixed[name]
    if name.startswith("pool."):
        leaf = name[5:]
        if leaf.startswith("norm_"):  # norm_q_w -> norm1_q.weight
            return f"{ve}clip_projector.norm1_{leaf[5]}.{'weight' if leaf.endswith('_w') else 'bias'}"
        x = leaf[0]  # q_w -> cross_attn.q.weight, q_b -> cross_attn.q_bias
        return f"{ve}clip_projector.cross_attn.{x}.weight" if leaf.endswith("_w") else f"{ve}clip_projector.cross_attn.{x}_bias"
    layer, leaf = name[1:].split(".", 1)
    b = f"{ve}blocks.{layer}."
    return b + {"norm1_w": "norm1.weight", "qkv_w": "attn.qkv.weight", "q_norm_w": "attn.q_norm.weight", "k_norm_w": "attn.k_norm.weight",
                "proj_w": "attn.proj.weight", "proj_b": "attn.proj.bias", "ls1": "ls1.gamma", "norm2_w": "norm2.weight",
                "fc1_w": "mlp.fc1.weight", "fc1_b": "mlp.fc1.bias", "fc2_w": "mlp.fc2.weight", "fc2_b": "mlp.fc2.bias", "ls2": "ls2.gamma"}[leaf]  # fmt: skip


def tensor_shapes(cfg: dict) -> dict[str, tuple[int, ...]]:
    """Shape of every tower tensor, in cb_iv2_set_tensor's names."""
    d, m = cfg["hidden"], cfg["mlp"]
    tokens = cfg["frames"] * (cfg["image_size"] // cfg["patch"]) ** 2 + 1
    s = {"patch_w": (d, 3 * cfg["patch"] ** 2), "patch_b": (d,), "cls": (d,), "pos": (tokens, d)}
    for i in range(cfg["layers"]):
        p = f"L{i}."
        s.update({p + "norm1_w": (d,), p + "qkv_w": (3 * d, d), p + "q_norm_w": (d,), p + "k_norm_w": (d,), p + "proj_w": (d, d),
                  p + "proj_b": (d,), p + "ls1": (d,), p + "norm2_w": (d,), p + "fc1_w": (m, d), p + "fc1_b": (m,), p + "fc2_w": (d, m),
                  p + "fc2_b": (d,), p + "ls2": (d,)})  # fmt: skip
    for x in "qkv":
        s.update({f"pool.norm_{x}_w": (d,), f"pool.norm_{x}_b": (d,), f"pool.{x}_w": (d, d), f"pool.{x}_b": (d,)})
    c, e = cfg["clip_dim"], cfg["embed_dim"]
    s.update({"pool.proj_w": (c, d), "pool.proj_b": (c,), "vproj_w": (e, c), "vproj_b": (e,)})
    return s


def seeded_weights(cfg: dict, seed: int, gamma=(0.05, 1.5)) -> dict[str, np.ndarray]:
    """Seeded float32 weights in the tower's names (numpy.random.default_rng(seed), drawn in tensor_shapes order).  Linear weights
    ~ N(0, 1/fan_in) (activations stay O(1) through the depth); norm weights ~ 1 + U(-0.2, 0.2), biases ~ N(0, 0.02^2) and
    LayerNorm biases ~ N(0, 0.1^2) - all nonzero; pos ~ N(0, 0.02^2), cls ~ N(0, 0.02^2) as trunc_normal_ draws them.  `gamma`: a
    (lo, hi) range for the LayerScale gammas (uniform) or one constant (1e-5 is the reference's init value)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in tensor_shapes(cfg).items():
        leaf = name.split(".")[-1]
        if leaf in ("ls1", "ls2"):
            a = rng.uniform(gamma[0], gamma[1], shape) if isinstance(gamma, tuple) else np.full(shape, gamma)
        elif "norm" in leaf and leaf.endswith("_w"):
            a = 1.0 + rng.uniform(-0.2, 0.2, shape)
        elif leaf.startswith("norm_") and leaf.endswith("_b"):
            a = rng.normal(0, 0.1, shape)
        elif len(shape) == 2 and name != "pos":
            a = rng.normal(0, 1.0 / math.sqrt(shape[1]), shape)
        else:
            a = rng.normal(0, 0.02, shape)
        out[name] = a.astype(np.float32)
    return out


def text_reference_keys(name: str) -> list[str]:
    """The reference checkpoint keys of text tower tensor `name` (cb_iv2_text_set_tensor's names), concatenated along dim 0 in this
    order (query | key | value for the fused QKV); type_emb is row 0 of the first key."""
    emb = "text_encoder.bert.embeddings."
    fixed = {"tok_emb": emb + "word_embeddings.weight", "pos_emb": emb + "position_embeddings.weight", "type_emb": emb + "token_type_embeddings.weight",
             "emb_ln_w": emb + "LayerNorm.weight", "emb_ln_b": emb + "LayerNorm.bias", "tproj_w": "text_proj.weight", "tproj_b": "text_proj.bias"}  # fmt: skip
    if name in fixed:
        return [fixed[name]]
    layer, leaf = name[1:].split(".", 1)
    b = f"text_encoder.bert.encoder.layer.{layer}."
    wb = "weight" if leaf.endswith("_w") else "bias"
    if leaf.startswith("qkv_"):
        return [f"{b}attention.self.{x}.{wb}" for x in ("query", "key", "value")]
    return [b + {"proj": "attention.output.dense", "ln1": "attention.output.LayerNorm", "fc1": "intermediate.dense", "fc2": "output.dense",
                 "ln2": "output.LayerNorm"}[leaf[:-2]] + "." + wb]  # fmt: skip


def text_tensor_shapes(cfg: dict) -> dict[str, tuple[int, ...]]:
    """Shape of every text tower tensor, in cb_iv2_text_set_tensor's names."""
    d, m = cfg["hidden"], cfg["mlp"]
    s = {"tok_emb": (cfg["vocab"], d), "pos_emb": (cfg["max_pos"], d), "type_emb": (d,), "emb_ln_w": (d,), "emb_ln_b": (d,)}
    for i in range(cfg["layers"]):
        p = f"L{i}."
        s.update({p + "qkv_w": (3 * d, d), p + "qkv_b": (3 * d,), p + "proj_w": (d, d), p + "proj_b": (d,), p + "ln1_w": (d,), p + "ln1_b": (d,),
                  p + "fc1_w": (m, d), p + "fc1_b": (m,), p + "fc2_w": (d, m), p + "fc2_b": (d,), p + "ln2_w": (d,), p + "ln2_b": (d,)})  # fmt: skip
    s.update({"tproj_w": (cfg["embed_dim"], d), "tproj_b": (cfg["embed_dim"],)})
    return s


def seeded_text_weights(cfg: dict, seed: int) -> dict[str, np.ndarray]:
    """Seeded float32 text tower weights (numpy.random.default_rng(seed), drawn in text_tensor_shapes order).  Linear weights
    ~ N(0, 1/fan_in), embeddings ~ N(0, 1), LayerNorm weights ~ 1 + U(-0.2, 0.2), biases ~ N(0, 0.02^2), LayerNorm biases ~ N(0, 0.1^2)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in text_tensor_shapes(cfg).items():
        leaf = name.split(".")[-1]
        if leaf in ("tok_emb", "pos_emb", "type_emb"):
            a = rng.normal(0, 1.0, shape)
        elif leaf.endswith("ln_w") or leaf in ("ln1_w", "ln2_w"):
            a = 1.0 + rng.uniform(-0.2, 0.2, shape)
        elif leaf.endswith("ln_b") or leaf in ("ln1_b", "ln2_b"):
            a = rng.normal(0, 0.1, shape)
        elif len(shape) == 2:
            a = rng.normal(0, 1.0 / math.sqrt(shape[1]), shape)
        else:
            a = rng.normal(0, 0.02, shape)
        out[name] = a.astype(np.float32)
    return out


def frames_of_pos_embed(pos_embed_shape, image_size: int = 224, patch: int = 14) -> int:
    """Frame count a pos_embed [1, T * g^2 + 1, d] was trained for."""
    g2 = (image_size // patch) ** 2
    tokens = int(pos_embed_shape[-2])
    if (tokens - 1) % g2:
        msg = f"pos_embed with {tokens} tokens is not [CLS] + frames x {g2} patches"
        raise ValueError(msg)
    return (tokens - 1) // g2


def _state_dict(path: str | Path) -> dict:
    sd = torch.load(os.fspath(path), map_location="cpu", weights_only=True)
    for key in ("model", "module"):
        if isinstance(sd, dict) and key in sd and isinstance(sd[key], dict):
            return sd[key]
    return sd


def load_text_checkpoint(path: str | Path, cfg: dict) -> dict[str, np.ndarray]:
    """The reference's .pt -> the text tower's float32 tensors (first cfg["layers"] encoder layers).  A missing key raises KeyError
    naming it; a tensor of the wrong size raises ValueError."""
    sd = _state_dict(path)
    out = {}
    for name, shape in text_tensor_shapes(cfg).items():
        parts = []
        for key in text_reference_keys(name):
            if key not in sd:
                msg = f"checkpoint {path} has no {key} (text tower tensor {name})"
                raise KeyError(msg)
            parts.append(sd[key].detach().float().cpu().reshape(-1, *sd[key].shape[1:]))
        a = torch.cat(parts, 0).numpy()
        if name == "type_emb":
            a = a[0]  # token type 0
        if a.size != math.prod(shape):
            msg = f"checkpoint tensor for {name} has shape {tuple(a.shape)}, the text tower takes {shape}"
            raise ValueError(msg)
        out[name] = np.ascontiguousarray(a.reshape(shape), dtype=np.float32)
    return out


def load_checkpoint(path: str | Path, cfg: dict) -> dict[str, np.ndarray]:
    """The reference's .pt -> the tower's float32 tensors.  A checkpoint whose pos_embed frame count differs from cfg["frames"] is
    refused (interpolate_pos_embed_internvideo2_new is the identity only when the counts match)."""
    sd = _state_dict(path)
    pos = sd["vision_encoder.pos_embed"]
    t = frames_of_pos_embed(pos.shape, cfg["image_size"], cfg["patch"])
    if t != cfg["frames"]:
        msg = f"checkpoint pos_embed is for {t} frames, the tower takes {cfg['frames']}"
        raise ValueError(msg)
    out = {}
    for name in tensor_shapes(cfg):
        a = sd[reference_key(name)].detach().float().cpu().numpy()
        if name == "patch_w":  # Conv3d [hidden, 3, 1, p, p] -> [hidden, 3 p^2], k = (c, y, x)
            a = a.reshape(a.shape[0], -1)
        elif name in ("cls", "pos"):
            a = a.reshape(-1, cfg["hidden"]) if name == "pos" else a.reshape(cfg["hidden"])
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def _find_checkpoint(d: Path) -> Path:
    for cand in (d / CHECKPOINT_NAME, *sorted(d.glob("*.pt"))):
        if cand.is_file():
            return cand
    msg = f"no {CHECKPOINT_NAME} (or other .pt) under {d}"
    raise FileNotFoundError(msg)


class InternVideo2MultiModality(ModelInterface):
    def __init__(self, *, weights_dir: str | Path | None = None, checkpoint: str | Path | None = None, seed: int | None = None,
                 max_clips: int = 8, config: dict | None = None, text_config: dict | None = None, vocab_file: str | Path | None = None,
                 max_texts: int = 64) -> None:  # fmt: skip
        super().__init__()
        self._weights_dir, self._checkpoint, self._seed, self._max_clips = weights_dir, checkpoint, seed, max_clips
        self._cfg = dict(config or IV2_1B_CFG)
        self._text_cfg = dict(text_config or IV2_TEXT_CFG)
        self._vocab_file, self._max_texts = vocab_file, max_texts
        self._weights: dict | None = None
        self._tower: Iv2Tower | None = None
        self._text_tower: Iv2TextTower | None = None
        self._tokenizer: BertTokenizer | None = None

    @property
    def conda_env_name(self) -> str:
        return "unified"

    @property
    def model_id_names(self) -> list[str]:
        return [_IV2_MODEL_ID]

    def _checkpoint_path(self) -> Path | None:
        if self._checkpoint is not None:
            return Path(self._checkpoint)
        d = src.resolve_dir(self.model_id_names[0], self._weights_dir)
        return _find_checkpoint(d) if d is not None else None

    def _missing_weights(self) -> FileNotFoundError:
        return FileNotFoundError(f"weights for {self.model_id_names[0]} not found (reference weight cache, CURATE_B200_WEIGHTS_DIR) and "
                                 "synthetic weights were not requested (seed= / CURATE_B200_SYNTHETIC_WEIGHTS)")  # fmt: skip

    def _load_weights(self) -> dict:
        if self._weights is not None:
            return self._weights
        path = self._checkpoint_path()
        if path is not None:
            with torch.serialization.safe_globals([set]):  # the reference adds `set` too (internvideo2.py:727)
                self._weights = load_checkpoint(path, self._cfg)
        else:
            seed = src.synthetic_seed(self._seed)
            if seed is None:
                raise self._missing_weights()
            self._weights = seeded_weights(self._cfg, seed)
        return self._weights

    def setup(self) -> None:
        if self._tower is not None:
            return
        self._tower = Iv2Tower(get_context(), self._cfg, self._load_weights(), max_clips=self._max_clips)

    def get_target_num_frames(self) -> int:
        """Frames per tube, read from the checkpoint's pos_embed (4 for InternVideo2-stage2_1b-224p-f4.pt)."""
        w = self._load_weights()
        return frames_of_pos_embed((1, *w["pos"].shape), self._cfg["image_size"], self._cfg["patch"])

    @property
    def tower(self) -> Iv2Tower:
        assert self._tower is not None, "setup() was not called"
        return self._tower

    def encode_batched_videos(self, videos: list[np.ndarray], batch_size: int) -> list[np.ndarray]:
        """videos: float32 tubes [1, T, 3, 224, 224] (or [T, 3, 224, 224]) -> one unit-norm float32 [1, embed_dim] per video.
        A tube whose frame count differs from the tower's raises ValueError (the reference fails there too, on the pos_embed add)."""
        tower = self.tower
        s = self._cfg["image_size"]
        tubes = []
        for v in videos:
            a = np.asarray(v, dtype=np.float32)
            a = a[0] if a.ndim == 5 and a.shape[0] == 1 else a
            if a.ndim != 4 or tuple(a.shape[1:]) != (3, s, s):
                msg = f"expected a tube [1, T, 3, {s}, {s}], got {np.shape(v)}"
                raise ValueError(msg)
            if a.shape[0] != tower.frames:
                msg = f"tube has {a.shape[0]} frames, the InternVideo2 tower takes {tower.frames}"
                raise ValueError(msg)
            tubes.append(a)
        out: list[np.ndarray] = []
        dev = f"cuda:{tower.ctx.device}"
        for i in range(0, len(tubes), max(1, batch_size)):
            batch = torch.from_numpy(np.stack(tubes[i : i + max(1, batch_size)])).to(dev)
            emb = tower.forward(batch).cpu().numpy()
            out += [e[None].copy() for e in emb]
        return out

    # ---- text side ---------------------------------------------------------------------------------------------------------
    @property
    def tokenizer(self) -> BertTokenizer:
        """google-bert/bert-large-uncased's vocab.txt (vocab_file=, else the reference weight cache / CURATE_B200_WEIGHTS_DIR)."""
        if self._tokenizer is None:
            path = Path(self._vocab_file) if self._vocab_file is not None else None
            if path is None:
                d = src.resolve_dir(BERT_VOCAB_ID, None)
                path = d / "vocab.txt" if d is not None else None
            if path is None or not path.is_file():
                msg = f"vocab.txt of {BERT_VOCAB_ID} not found (vocab_file=, reference weight cache, CURATE_B200_WEIGHTS_DIR)"
                raise FileNotFoundError(msg)
            tok = BertTokenizer.from_file(path)
            if len(tok.vocab) > self._text_cfg["vocab"]:
                msg = f"{path} has {len(tok.vocab)} tokens, the text tower embeds {self._text_cfg['vocab']}"
                raise ValueError(msg)
            self._tokenizer = tok
        return self._tokenizer

    def setup_text(self) -> None:
        """Builds the text tower (about 0.5 GB of BERT weights on the GPU); the text methods call it on first use."""
        if self._text_tower is not None:
            return
        tok = self.tokenizer
        path = self._checkpoint_path()
        if path is not None:
            weights = load_text_checkpoint(path, self._text_cfg)
        else:
            seed = src.synthetic_seed(self._seed)
            if seed is None:
                raise self._missing_weights()
            weights = seeded_text_weights(self._text_cfg, seed)
        self._text_tower = Iv2TextTower(get_context(), self._text_cfg, weights, max_texts=self._max_texts, max_len=MAX_TXT_L)
        self._tokenizer = tok

    def encode_texts(self, texts: list[str]) -> np.ndarray:
        """Captions -> unit-norm float32 [n, embed_dim] (get_txt_feat per text, internvideo2_mm.py:219-241, batched: a text's
        embedding does not depend on the others)."""
        if not texts:
            return np.zeros((0, self._text_cfg["embed_dim"]), dtype=np.float32)
        self.setup_text()
        ids, lengths = self.tokenizer(list(texts), MAX_TXT_L)
        return self._text_tower.forward(ids, lengths).cpu().numpy()

    def get_text_embedding(self, text: str) -> torch.Tensor:
        """One caption -> float32 [1, embed_dim] (InternVideo2MultiModality.get_text_embedding, internvideo2_mm.py:481-492)."""
        return torch.from_numpy(self.encode_texts([text]))

    @staticmethod
    def evaluate(video_embd, text_embds) -> tuple[list[float], list[int]]:
        """softmax(100 * v . t^T) over the texts in float32, all of them ranked (InternVideo2MultiModality.evaluate /
        predict_label, internvideo2_mm.py:243-254, :494-511): (probabilities, text indices), most probable first, ties to the
        lower index.  video_embd [1, d]; text_embds a list of [1, d] (or an array [n, d])."""
        v = torch.as_tensor(np.asarray(video_embd, dtype=np.float32)).reshape(1, -1)
        t = torch.as_tensor(np.concatenate([np.asarray(x, dtype=np.float32).reshape(-1, v.shape[1]) for x in text_embds], 0))
        probs = (100.0 * v @ t.T).softmax(dim=-1)[0].numpy()
        order = np.argsort(-probs, kind="stable")
        return probs[order].tolist(), order.tolist()
