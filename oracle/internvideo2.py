"""InternVideo2-1B clip embedding (the vision half of InternVideo2_Stage2.get_vid_feat, models/internvideo2_mm.py:203-217) restated
in torch: PretrainInternVideo2.forward (internvideo2.py:596-650) up to clip_projector, vision_proj, L2 norm.  Weights use the tower's
names (include/curate_b200.h, cb_iv2_set_tensor); cosmos_curate_b200.models.internvideo2 maps the reference's checkpoint keys onto them.

Runs in any dtype on any device: float32 on the CPU is what the golden vectors pin, float32 on the GPU what the full-depth test
compares with, bf16 on the GPU the library-path baseline of tools/prof_iv2.py (the precision the reference runs at).
Test infrastructure only (see oracle/__init__.py); it never reads the reference checkout.
"""

from __future__ import annotations

from dataclasses import asdict, dataclass, replace

import numpy as np
import torch
import torch.nn.functional as F

MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)  # internvideo2_mm.py:378-379
STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)


@dataclass(frozen=True)
class Iv2Config:
    image_size: int = 224
    patch: int = 14
    frames: int = 4
    hidden: int = 1408
    layers: int = 40
    heads: int = 16
    mlp: int = 6144
    clip_dim: int = 768
    embed_dim: int = 512
    rms_eps: float = 1e-6
    ln_eps: float = 1e-5

    @property
    def tokens(self) -> int:
        return self.frames * (self.image_size // self.patch) ** 2 + 1

    def to_dict(self) -> dict:
        return asdict(self)

    def with_(self, **kw) -> "Iv2Config":
        return replace(self, **kw)


IV2_1B = Iv2Config()  # pretrain_internvideo2_1b_patch14_224 with the shipped config (num_frames 4, clip_embed_dim 768, embed_dim 512)


def flops_per_clip(cfg: Iv2Config) -> float:
    """2 M N K of the block GEMMs plus 4 T^2 d heads of attention, over all layers (the patch embed and the pooling are not counted):
    2.31e12 for the 1B tower at 4 frames."""
    t, d, m = cfg.tokens, cfg.hidden, cfg.mlp
    per_layer = 2 * t * d * (3 * d) + 2 * t * d * d + 2 * 2 * t * d * m + 4 * t * t * (d // cfg.heads) * cfg.heads
    return float(per_layer * cfg.layers)


def random_weights(cfg: Iv2Config, seed: int, gamma=(0.05, 1.5)) -> dict[str, np.ndarray]:
    """The tower's seeded weights (cosmos_curate_b200.models.internvideo2.seeded_weights) for this config."""
    from cosmos_curate_b200.models.internvideo2 import seeded_weights

    return seeded_weights(cfg.to_dict(), seed, gamma)


def expand_frames(frames_u8: np.ndarray, block: int) -> np.ndarray:
    """uint8 [..., H, W, 3] -> [..., H * block, W * block, 3]: every pixel repeated into a block x block square."""
    return np.repeat(np.repeat(frames_u8, block, axis=-3), block, axis=-2)


def tube_from_frames(frames_u8: np.ndarray) -> np.ndarray:
    """uint8 [..., T, H, W, 3] RGB -> float32 [..., T, 3, H, W]: ((x / 255 - mean) / std), the tube formulation of
    internvideo2_mm.py:385-405 (frames already at the tower's size)."""
    x = (frames_u8.astype(np.float32) / np.float32(255.0) - MEAN) / STD
    return np.ascontiguousarray(np.moveaxis(x, -1, -3))


def _rms(x, w, eps):
    xf = x.float()
    return (w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))).to(x.dtype)


def forward(cfg: Iv2Config, w: dict, tubes, dtype=torch.float32, device="cpu") -> torch.Tensor:
    """tubes float32 [n][T][3][S][S] -> unit-norm embeddings [n][embed_dim] (float32)."""
    W = {k: (torch.as_tensor(v).to(device=device, dtype=dtype)) for k, v in w.items()}
    x = torch.as_tensor(tubes).to(device=device, dtype=dtype)
    n, t = x.shape[:2]
    assert t == cfg.frames, (t, cfg.frames)
    d, h, p = cfg.hidden, cfg.heads, cfg.patch
    hd = d // h
    g = cfg.image_size // p
    # Conv3d(k = (1, p, p), stride = kernel) as patches . W^T; tokens ordered t * g^2 + (row * g + col)
    patches = x.reshape(n, t, 3, g, p, g, p).permute(0, 1, 3, 5, 2, 4, 6).reshape(n, t * g * g, 3 * p * p)
    z = patches @ W["patch_w"].T + W["patch_b"]
    z = torch.cat([W["cls"].expand(n, 1, d), z], dim=1) + W["pos"]
    for i in range(cfg.layers):
        L = lambda k: W[f"L{i}.{k}"]  # noqa: E731
        y = _rms(z, L("norm1_w"), cfg.rms_eps)
        qkv = y @ L("qkv_w").T
        q, k, v = qkv.split(d, dim=-1)
        q, k = _rms(q, L("q_norm_w"), cfg.rms_eps), _rms(k, L("k_norm_w"), cfg.rms_eps)
        q, k, v = (a.reshape(n, -1, h, hd).transpose(1, 2) for a in (q, k, v))
        a = F.scaled_dot_product_attention(q, k, v, scale=hd**-0.5).transpose(1, 2).reshape(n, -1, d)
        a = a @ L("proj_w").T + L("proj_b")
        z = z + (a.float() * L("ls1").float()).to(z.dtype)
        y = _rms(z, L("norm2_w"), cfg.rms_eps)
        y = F.gelu(y @ L("fc1_w").T + L("fc1_b")) @ L("fc2_w").T + L("fc2_b")
        z = z + (y.float() * L("ls2").float()).to(z.dtype)
    # clip_projector: AttentionPoolingBlock, one query per clip
    ln = lambda a, x_: F.layer_norm(a, (d,), W[f"pool.norm_{x_}_w"], W[f"pool.norm_{x_}_b"], cfg.ln_eps)  # noqa: E731
    xq = ln(z.mean(1, keepdim=True), "q")
    q = (xq @ W["pool.q_w"].T + W["pool.q_b"]).reshape(n, 1, h, hd).transpose(1, 2)
    k = (ln(z, "k") @ W["pool.k_w"].T + W["pool.k_b"]).reshape(n, -1, h, hd).transpose(1, 2)
    v = (ln(z, "v") @ W["pool.v_w"].T + W["pool.v_b"]).reshape(n, -1, h, hd).transpose(1, 2)
    att = torch.softmax((q * hd**-0.5) @ k.transpose(-1, -2), dim=-1)
    pooled = (att @ v).transpose(1, 2).reshape(n, d) @ W["pool.proj_w"].T + W["pool.proj_b"]
    e = (pooled @ W["vproj_w"].T + W["vproj_b"]).float()
    return e / e.norm(dim=-1, keepdim=True)
