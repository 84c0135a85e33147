"""Tower configurations and weight sources (host side).

* `VitConfig` + the three configurations BASELINE.json names (CLIP ViT-L/14 is the reference's only CLIP,
  cosmos_curate/models/clip.py:33; ViT-B/32 and SigLIP SoViT-400m are served by the same tower).
* `load_hf_clip_dir` reads a Hugging Face `CLIPModel` checkpoint directory (what the reference passes to
  `CLIPModel.from_pretrained`, clip.py:40-41) without instantiating the torch model.
* `load_aesthetic_mlp` reads the reference's aesthetic head checkpoint (aesthetics.py:77-82: `model.safetensors`
  with keys `layers.{0,2,4,6,7}.{weight,bias}`) and folds it to one affine map - the MLP has no non-linearity.
* `seeded_weights` produces deterministic random weights for synthetic benchmarks (no checkpoints offline).
"""

from __future__ import annotations

import json
from dataclasses import asdict, dataclass
from pathlib import Path

import numpy as np


@dataclass(frozen=True)
class VitConfig:
    image_size: int = 224
    patch: int = 14
    hidden: int = 1024
    layers: int = 24
    heads: int = 16
    mlp: int = 4096
    proj_dim: int = 768
    act: str = "quick_gelu"
    ln_eps: float = 1e-5
    arch: str = "clip"

    @property
    def tokens(self) -> int:
        g = self.image_size // self.patch
        return g * g + (1 if self.arch == "clip" else 0)

    def to_dict(self) -> dict:
        return asdict(self)

    def flops_per_image(self) -> float:
        """2*M*N*K over patch-embed, QKV, QK^T, PV, out-proj, MLP and projection (SURVEY.md 8d)."""
        t, d, m = self.tokens, self.hidden, self.mlp
        g2 = (self.image_size // self.patch) ** 2
        per_layer = 2 * t * d * 3 * d + 2 * t * d * d + 2 * 2 * t * t * d + 2 * 2 * t * d * m
        return self.layers * per_layer + 2 * g2 * 3 * self.patch**2 * d + 2 * d * self.proj_dim

    def gemm_flops_per_image(self) -> float:
        """The part executed by the wgmma GEMM kernel (everything but attention's QK^T / PV and the pooled tail)."""
        t, d, m = self.tokens, self.hidden, self.mlp
        g2 = (self.image_size // self.patch) ** 2
        return self.layers * (2 * t * d * 3 * d + 2 * t * d * d + 2 * 2 * t * d * m) + 2 * g2 * 3 * self.patch**2 * d


CLIP_VIT_L14 = VitConfig()
CLIP_VIT_B32 = VitConfig(patch=32, hidden=768, layers=12, heads=12, mlp=3072, proj_dim=512)
SIGLIP_SO400M_384 = VitConfig(image_size=384, patch=14, hidden=1152, layers=27, heads=16, mlp=4304, proj_dim=0, act="gelu_tanh", ln_eps=1e-6, arch="siglip")
CONFIGS = {"clip-vit-large-patch14": CLIP_VIT_L14, "clip-vit-base-patch32": CLIP_VIT_B32, "siglip-so400m-patch14-384": SIGLIP_SO400M_384}

AESTHETIC_LINEAR_KEYS = ("layers.0", "layers.2", "layers.4", "layers.6", "layers.7")


def seeded_weights(cfg: VitConfig, seed: int = 0) -> dict[str, np.ndarray]:
    rng = np.random.default_rng(seed)
    d, m, kp = cfg.hidden, cfg.mlp, 3 * cfg.patch * cfg.patch

    def rn(*shape, std):
        return (rng.standard_normal(shape, dtype=np.float32) * np.float32(std)).astype(np.float32)

    w = {"patch_w": rn(d, kp, std=kp**-0.5), "pos": rn(cfg.tokens, d, std=0.02)}
    if cfg.arch == "clip":
        w.update(cls=rn(d, std=0.02), pre_ln_w=1 + rn(d, std=0.05), pre_ln_b=rn(d, std=0.02))
    else:
        w["patch_b"] = rn(d, std=0.02)
    res = (2 * cfg.layers) ** -0.5
    for i in range(cfg.layers):
        p = f"L{i}."
        w[p + "ln1_w"], w[p + "ln1_b"] = 1 + rn(d, std=0.05), rn(d, std=0.02)
        w[p + "qkv_w"], w[p + "qkv_b"] = rn(3 * d, d, std=d**-0.5), rn(3 * d, std=0.02)
        w[p + "out_w"], w[p + "out_b"] = rn(d, d, std=d**-0.5 * res), rn(d, std=0.02)
        w[p + "ln2_w"], w[p + "ln2_b"] = 1 + rn(d, std=0.05), rn(d, std=0.02)
        w[p + "fc1_w"], w[p + "fc1_b"] = rn(m, d, std=d**-0.5), rn(m, std=0.02)
        w[p + "fc2_w"], w[p + "fc2_b"] = rn(d, m, std=m**-0.5 * res), rn(d, std=0.02)
    w["post_ln_w"], w["post_ln_b"] = 1 + rn(d, std=0.05), rn(d, std=0.02)
    if cfg.proj_dim:
        w["proj_w"] = rn(cfg.proj_dim, d, std=d**-0.5)
    if cfg.arch == "siglip":  # MAP pooling head (HF SiglipMultiheadAttentionPoolingHead)
        w.update(map_probe=rn(d, std=0.02), map_in_w=rn(3 * d, d, std=d**-0.5), map_in_b=rn(3 * d, std=0.02), map_out_w=rn(d, d, std=d**-0.5),
                 map_out_b=rn(d, std=0.02), map_ln_w=1 + rn(d, std=0.05), map_ln_b=rn(d, std=0.02), map_fc1_w=rn(m, d, std=d**-0.5),
                 map_fc1_b=rn(m, std=0.02), map_fc2_w=rn(d, m, std=m**-0.5), map_fc2_b=rn(d, std=0.02))  # fmt: skip
    return w


def seeded_aesthetic(dim: int, seed: int = 0) -> tuple[np.ndarray, float]:
    rng = np.random.default_rng(10_000 + seed)
    return (rng.standard_normal(dim, dtype=np.float32) * np.float32(dim**-0.5 * 4)).astype(np.float32), 5.0


def fold_aesthetic_mlp(state: dict[str, np.ndarray]) -> tuple[np.ndarray, float]:
    """Activation-free 5-layer MLP -> (w, b) with score = w . e + b; folded in float64."""
    a, b = None, None
    for k in AESTHETIC_LINEAR_KEYS:
        wk, bk = state[k + ".weight"].astype(np.float64), state[k + ".bias"].astype(np.float64)
        a = wk if a is None else wk @ a
        b = bk if b is None else wk @ b + bk
    return a.reshape(-1).astype(np.float32), float(b.reshape(-1)[0])


def load_aesthetic_mlp(path: str | Path) -> tuple[np.ndarray, float]:
    from safetensors.numpy import load_file

    return fold_aesthetic_mlp(load_file(str(path)))


def _hf_state(model_dir: Path) -> dict[str, np.ndarray]:
    from safetensors.numpy import load_file

    files = sorted(model_dir.glob("*.safetensors"))
    if not files:
        msg = f"no *.safetensors under {model_dir}"
        raise FileNotFoundError(msg)
    sd: dict[str, np.ndarray] = {}
    for f in files:
        sd.update(load_file(str(f)))
    return sd


def weights_from_hf_clip_state(sd: dict[str, np.ndarray], cfg: VitConfig) -> dict[str, np.ndarray]:
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    v = "vision_model."
    w = {
        "patch_w": f32(sd[v + "embeddings.patch_embedding.weight"]).reshape(cfg.hidden, -1),
        "cls": f32(sd[v + "embeddings.class_embedding"]),
        "pos": f32(sd[v + "embeddings.position_embedding.weight"]),
        "pre_ln_w": f32(sd[v + "pre_layrnorm.weight"]), "pre_ln_b": f32(sd[v + "pre_layrnorm.bias"]),
        "post_ln_w": f32(sd[v + "post_layernorm.weight"]), "post_ln_b": f32(sd[v + "post_layernorm.bias"]),
        "proj_w": f32(sd["visual_projection.weight"]),
    }  # fmt: skip
    for i in range(cfg.layers):
        s, p = f"{v}encoder.layers.{i}.", f"L{i}."
        w[p + "ln1_w"], w[p + "ln1_b"] = f32(sd[s + "layer_norm1.weight"]), f32(sd[s + "layer_norm1.bias"])
        w[p + "ln2_w"], w[p + "ln2_b"] = f32(sd[s + "layer_norm2.weight"]), f32(sd[s + "layer_norm2.bias"])
        w[p + "qkv_w"] = np.concatenate([f32(sd[s + f"self_attn.{n}_proj.weight"]) for n in "qkv"], axis=0)
        w[p + "qkv_b"] = np.concatenate([f32(sd[s + f"self_attn.{n}_proj.bias"]) for n in "qkv"], axis=0)
        w[p + "out_w"], w[p + "out_b"] = f32(sd[s + "self_attn.out_proj.weight"]), f32(sd[s + "self_attn.out_proj.bias"])
        w[p + "fc1_w"], w[p + "fc1_b"] = f32(sd[s + "mlp.fc1.weight"]), f32(sd[s + "mlp.fc1.bias"])
        w[p + "fc2_w"], w[p + "fc2_b"] = f32(sd[s + "mlp.fc2.weight"]), f32(sd[s + "mlp.fc2.bias"])
    return w


def load_hf_clip_dir(model_dir: str | Path) -> tuple[VitConfig, dict[str, np.ndarray]]:
    model_dir = Path(model_dir)
    c = json.loads((model_dir / "config.json").read_text())
    vc = c.get("vision_config", c)
    cfg = VitConfig(
        image_size=vc.get("image_size", 224), patch=vc.get("patch_size", 32), hidden=vc.get("hidden_size", 768),
        layers=vc.get("num_hidden_layers", 12), heads=vc.get("num_attention_heads", 12), mlp=vc.get("intermediate_size", 3072),
        proj_dim=c.get("projection_dim", vc.get("projection_dim", 512)), act=vc.get("hidden_act", "quick_gelu"),
        ln_eps=vc.get("layer_norm_eps", 1e-5), arch="clip",
    )  # fmt: skip
    return cfg, weights_from_hf_clip_state(_hf_state(model_dir), cfg)


def weights_from_hf_siglip_state(sd: dict[str, np.ndarray], cfg: VitConfig) -> dict[str, np.ndarray]:
    """transformers SiglipVisionModel / SiglipModel state dict (vision side) -> tower tensor names."""
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    v = "vision_model."
    w = {
        "patch_w": f32(sd[v + "embeddings.patch_embedding.weight"]).reshape(cfg.hidden, -1), "patch_b": f32(sd[v + "embeddings.patch_embedding.bias"]),
        "pos": f32(sd[v + "embeddings.position_embedding.weight"]),
        "post_ln_w": f32(sd[v + "post_layernorm.weight"]), "post_ln_b": f32(sd[v + "post_layernorm.bias"]),
        "map_probe": f32(sd[v + "head.probe"]).reshape(-1),
        "map_in_w": f32(sd[v + "head.attention.in_proj_weight"]), "map_in_b": f32(sd[v + "head.attention.in_proj_bias"]),
        "map_out_w": f32(sd[v + "head.attention.out_proj.weight"]), "map_out_b": f32(sd[v + "head.attention.out_proj.bias"]),
        "map_ln_w": f32(sd[v + "head.layernorm.weight"]), "map_ln_b": f32(sd[v + "head.layernorm.bias"]),
        "map_fc1_w": f32(sd[v + "head.mlp.fc1.weight"]), "map_fc1_b": f32(sd[v + "head.mlp.fc1.bias"]),
        "map_fc2_w": f32(sd[v + "head.mlp.fc2.weight"]), "map_fc2_b": f32(sd[v + "head.mlp.fc2.bias"]),
    }  # fmt: skip
    for i in range(cfg.layers):
        s, p = f"{v}encoder.layers.{i}.", f"L{i}."
        w[p + "ln1_w"], w[p + "ln1_b"] = f32(sd[s + "layer_norm1.weight"]), f32(sd[s + "layer_norm1.bias"])
        w[p + "ln2_w"], w[p + "ln2_b"] = f32(sd[s + "layer_norm2.weight"]), f32(sd[s + "layer_norm2.bias"])
        w[p + "qkv_w"] = np.concatenate([f32(sd[s + f"self_attn.{n}_proj.weight"]) for n in "qkv"], axis=0)
        w[p + "qkv_b"] = np.concatenate([f32(sd[s + f"self_attn.{n}_proj.bias"]) for n in "qkv"], axis=0)
        w[p + "out_w"], w[p + "out_b"] = f32(sd[s + "self_attn.out_proj.weight"]), f32(sd[s + "self_attn.out_proj.bias"])
        w[p + "fc1_w"], w[p + "fc1_b"] = f32(sd[s + "mlp.fc1.weight"]), f32(sd[s + "mlp.fc1.bias"])
        w[p + "fc2_w"], w[p + "fc2_b"] = f32(sd[s + "mlp.fc2.weight"]), f32(sd[s + "mlp.fc2.bias"])
    return w


def load_hf_siglip_dir(model_dir: str | Path) -> tuple[VitConfig, dict[str, np.ndarray]]:
    """A Hugging Face SigLIP checkpoint directory (google/siglip-so400m-patch14-384 layout) without instantiating the torch model."""
    model_dir = Path(model_dir)
    c = json.loads((model_dir / "config.json").read_text())
    vc = c.get("vision_config", c)
    cfg = VitConfig(
        image_size=vc.get("image_size", 224), patch=vc.get("patch_size", 16), hidden=vc.get("hidden_size", 768),
        layers=vc.get("num_hidden_layers", 12), heads=vc.get("num_attention_heads", 12), mlp=vc.get("intermediate_size", 3072),
        proj_dim=0, act="gelu_tanh", ln_eps=vc.get("layer_norm_eps", 1e-6), arch="siglip",
    )  # fmt: skip
    return cfg, weights_from_hf_siglip_state(_hf_state(model_dir), cfg)
