"""InternVideo2 clip embeddings on the H100 path: the `ModelInterface` of the reference's InternVideo2MultiModality
(cosmos_curate/models/internvideo2_mm.py:306-479) for its vision side - `encode_batched_videos` returns one unit-norm float32
[1, 512] array per clip (InternVideo2_Stage2.get_vid_feat, :203-217, then np.split, :460-479).  The text tower (BERT) is not built.

Weights: the reference's checkpoint (InternVideo2-stage2_1b-224p-f4.pt, torch.load(weights_only=True), state dict under "model" or
"module"), of which the vision_encoder.* and vision_proj.* tensors are used; the text keys are ignored.  Seeded synthetic weights only
when explicitly requested (models/_weights_source.py).
"""

from __future__ import annotations

import math
import os
from pathlib import Path

import numpy as np
import torch

from ..interfaces import ModelInterface
from ..runtime import Iv2Tower, get_context
from . import _weights_source as src

_IV2_MODEL_ID = "OpenGVLab/InternVideo2-Stage2_1B-224p-f4"
CHECKPOINT_NAME = "InternVideo2-stage2_1b-224p-f4.pt"

# pretrain_internvideo2_1b_patch14_224 (internvideo2.py:696-735) with the shipped config (internvideo2_mm_config_model.json:390-461)
IV2_1B_CFG = {"image_size": 224, "patch": 14, "frames": 4, "hidden": 1408, "layers": 40, "heads": 16, "mlp": 6144, "clip_dim": 768,
              "embed_dim": 512, "rms_eps": 1e-6, "ln_eps": 1e-5}  # fmt: skip


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


def frames_of_pos_embed(pos_embed_shape, image_size: int = 224, patch: int = 14) -> int:
    """Frame count a pos_embed [1, T * g^2 + 1, d] was trained for."""
    g2 = (image_size // patch) ** 2
    tokens = int(pos_embed_shape[-2])
    if (tokens - 1) % g2:
        msg = f"pos_embed with {tokens} tokens is not [CLS] + frames x {g2} patches"
        raise ValueError(msg)
    return (tokens - 1) // g2


def load_checkpoint(path: str | Path, cfg: dict) -> dict[str, np.ndarray]:
    """The reference's .pt -> the tower's float32 tensors.  A checkpoint whose pos_embed frame count differs from cfg["frames"] is
    refused (interpolate_pos_embed_internvideo2_new is the identity only when the counts match)."""
    sd = torch.load(os.fspath(path), map_location="cpu", weights_only=True)
    for key in ("model", "module"):
        if isinstance(sd, dict) and key in sd and isinstance(sd[key], dict):
            sd = sd[key]
            break
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
                 max_clips: int = 8, config: dict | None = None) -> None:  # fmt: skip
        super().__init__()
        self._weights_dir, self._checkpoint, self._seed, self._max_clips = weights_dir, checkpoint, seed, max_clips
        self._cfg = dict(config or IV2_1B_CFG)
        self._weights: dict | None = None
        self._tower: Iv2Tower | None = None

    @property
    def conda_env_name(self) -> str:
        return "unified"

    @property
    def model_id_names(self) -> list[str]:
        return [_IV2_MODEL_ID]

    def _load_weights(self) -> dict:
        if self._weights is not None:
            return self._weights
        path = Path(self._checkpoint) if self._checkpoint is not None else None
        if path is None:
            d = src.resolve_dir(self.model_id_names[0], self._weights_dir)
            path = _find_checkpoint(d) if d is not None else None
        if path is not None:
            with torch.serialization.safe_globals([set]):  # the reference adds `set` too (internvideo2.py:727)
                self._weights = load_checkpoint(path, self._cfg)
        else:
            seed = src.synthetic_seed(self._seed)
            if seed is None:
                msg = (f"weights for {self.model_id_names[0]} not found (reference weight cache, CURATE_B200_WEIGHTS_DIR) and "
                       "synthetic weights were not requested (seed= / CURATE_B200_SYNTHETIC_WEIGHTS)")  # fmt: skip
                raise FileNotFoundError(msg)
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
