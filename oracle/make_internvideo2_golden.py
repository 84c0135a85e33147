"""Write tests/golden/internvideo2_ref.npz: the reference's own PretrainInternVideo2 (internvideo2.py, imported unmodified with a stub
`timm.layers`, see reference_vision_module) plus a vision_proj Linear, in float32 on the CPU, at the 1B tower's width (hidden 1408, 16 heads
of 88, mlp 6144) and depth 2, on seeded weights; and the same model in bf16 (the precision the reference runs at) on the same inputs.

Stored: the uint8 frames the tubes are formed from, at 1/7 of the tower's size (32 x 32; every pixel becomes a 7 x 7 block,
oracle.internvideo2.expand_frames, so each 14 x 14 patch holds 2 x 2 distinct values per channel and the file stays small), the
seeds, the gamma setting and the embeddings.  Tube = ((x / 255 - mean) / std), oracle.internvideo2.tube_from_frames.  The
weights are not stored: tests rebuild them with cosmos_curate_b200.models.internvideo2.seeded_weights(cfg, seed, gamma).

    python -m oracle.make_internvideo2_golden
"""

from __future__ import annotations

import importlib
import json
import sys
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from cosmos_curate_b200.models.internvideo2 import reference_key  # noqa: E402
from oracle import internvideo2 as O  # noqa: E402
from oracle import ref_import  # noqa: E402

FRAMES_SEED = 99
BLOCK = 7  # stored frames are 224 / BLOCK = 32 pixels square
# (name, frames, weight seed, gamma): LayerScale gammas drawn from U(0.05, 1.5), and at the reference's init value 1e-5
CASES = [("t4", 4, 11, (0.05, 1.5)), ("t8", 8, 12, (0.05, 1.5)), ("t4_init_gamma", 4, 13, 1e-5)]
DEPTH = 2


def golden_config(frames: int) -> O.Iv2Config:
    return O.IV2_1B.with_(frames=frames, layers=DEPTH)


def golden_frames() -> np.ndarray:
    """uint8 [2][8][32][32][3]: a seeded clip and its mirror image (two clips per case: a batch of two)."""
    a = np.random.default_rng(FRAMES_SEED).integers(0, 256, (8, 224 // BLOCK, 224 // BLOCK, 3), dtype=np.uint8)
    return np.stack([a, a[:, :, ::-1]])


def reference_vision_module():
    """The reference's own internvideo2.py (PretrainInternVideo2 and its blocks), imported with a stub `timm.layers` (timm is not
    installed): identity DropPath (drop_path is 0 in eval and the blocks skip it), to_2tuple, and trunc_normal_ (the module's
    initialisation only; every tensor is overwritten by reference_model), and `easydict` when it is missing.  The `av` and
    `model_utils` stubs are oracle/ref_import's."""
    ref_import._install_stubs()
    if "timm.layers" not in sys.modules:
        timm, layers = types.ModuleType("timm"), types.ModuleType("timm.layers")

        class DropPath(torch.nn.Identity):
            def __init__(self, *args, **kwargs):
                super().__init__()

        layers.DropPath = DropPath
        layers.to_2tuple = lambda x: tuple(x) if isinstance(x, (tuple, list)) else (x, x)
        layers.trunc_normal_ = lambda t, mean=0.0, std=1.0, a=-2.0, b=2.0: torch.nn.init.trunc_normal_(t, mean, std, a, b)
        timm.layers = layers
        sys.modules["timm"], sys.modules["timm.layers"] = timm, layers
    if "easydict" not in sys.modules:
        try:
            import easydict  # noqa: F401
        except ImportError:
            stub = types.ModuleType("easydict")
            stub.EasyDict = dict
            sys.modules["easydict"] = stub
    return importlib.import_module("cosmos_curate.models.internvideo2_multi_modality.internvideo2.internvideo2")


def reference_model(cfg: O.Iv2Config, w: dict):
    """PretrainInternVideo2 + vision_proj with the tower weights `w` loaded under the reference's own keys."""
    mod = reference_vision_module()
    model = mod.PretrainInternVideo2(in_chans=3, patch_size=cfg.patch, img_size=cfg.image_size, qkv_bias=False, drop_path_rate=0.0,
                                     embed_dim=cfg.hidden, num_heads=cfg.heads, mlp_ratio=48 / 11, init_values=1e-5, qk_normalization=True,
                                     depth=cfg.layers, attn_pool_num_heads=16, clip_embed_dim=cfg.clip_dim, layerscale_no_force_fp32=False,
                                     num_frames=cfg.frames, tubelet_size=1, sep_pos_embed=False, sep_image_video_pos_embed=False)  # fmt: skip
    assert model.blocks[0].mlp.fc1.out_features == cfg.mlp
    vision_proj = torch.nn.Linear(cfg.clip_dim, cfg.embed_dim)
    sd = model.state_dict()
    for name, a in w.items():
        key = reference_key(name)
        t = torch.from_numpy(a)
        if key.startswith("vision_proj."):
            getattr(vision_proj, key.split(".")[1]).data.copy_(t)
            continue
        key = key[len("vision_encoder.") :]
        assert key in sd, key
        sd[key] = t.reshape(sd[key].shape)
    model.load_state_dict(sd)
    return model.eval(), vision_proj.eval()


@torch.no_grad()
def reference_embeddings(model, vision_proj, tubes: np.ndarray, dtype) -> np.ndarray:
    """get_vid_feat (internvideo2_mm.py:203-217): vision_encoder(tube [B, 3, T, H, W])[1] -> vision_proj -> / norm."""
    model, vision_proj = model.to(dtype), vision_proj.to(dtype)
    x = torch.from_numpy(tubes).permute(0, 2, 1, 3, 4).to(dtype)
    e = vision_proj(model(x)[1]).float()
    return (e / e.norm(dim=-1, keepdim=True)).numpy()


def main() -> None:
    frames = golden_frames()
    out = {"frames_u8": frames, "meta": np.frombuffer(json.dumps({
        "frames_seed": FRAMES_SEED, "block": BLOCK, "depth": DEPTH, "cases": [{"name": n, "frames": t, "seed": s, "gamma": list(g) if isinstance(g, tuple) else g}
                                                             for n, t, s, g in CASES]}).encode(), dtype=np.uint8)}  # fmt: skip
    for name, t, seed, gamma in CASES:
        cfg = golden_config(t)
        w = O.random_weights(cfg, seed, gamma)
        tubes = O.tube_from_frames(O.expand_frames(frames[:, :t], BLOCK))
        model, vp = reference_model(cfg, w)
        out[f"{name}_emb"] = reference_embeddings(model, vp, tubes, torch.float32)
        out[f"{name}_emb_bf16"] = reference_embeddings(model, vp, tubes, torch.bfloat16)
        cos = (out[f"{name}_emb"] * out[f"{name}_emb_bf16"]).sum(-1)
        print(f"{name}: reference bf16 vs float32 cosine {cos.min():.6f}, max-abs {np.abs(out[f'{name}_emb'] - out[f'{name}_emb_bf16']).max():.2e}")
    path = ROOT / "tests" / "golden" / "internvideo2_ref.npz"
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({path.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
