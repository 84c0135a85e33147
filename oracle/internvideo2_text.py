"""InternVideo2 text embedding (InternVideo2_Stage2.get_txt_feat, models/internvideo2_mm.py:219-241, after tokenization) restated in
torch: BertModel(mode="text") (bert/xbert.py) - embeddings (word + token type 0 + position, LayerNorm), the first `layers` post-LN
self-attention layers with the padding mask, the [CLS] row, text_proj, L2 norm.  Weights use the text tower's names
(include/curate_b200.h, cb_iv2_text_set_tensor); cosmos_curate_b200.models.internvideo2 maps the reference's checkpoint keys onto them.

Runs in any dtype on any device: float32 on the CPU is what the golden vectors pin, float32 on the GPU what the full-depth test compares
with.  Test infrastructure only (see oracle/__init__.py); it never reads the reference checkout.
"""

from __future__ import annotations

from dataclasses import asdict, dataclass, replace

import numpy as np
import torch
import torch.nn.functional as F


@dataclass(frozen=True)
class TextConfig:
    hidden: int = 1024
    layers: int = 19
    heads: int = 16
    mlp: int = 4096
    vocab: int = 30522
    max_pos: int = 512
    embed_dim: int = 512
    ln_eps: float = 1e-12

    def to_dict(self) -> dict:
        return asdict(self)

    def with_(self, **kw) -> "TextConfig":
        return replace(self, **kw)


IV2_TEXT = TextConfig()  # BERT-large in mode="text": fusion_layer = 19 of its 24 layers, text_proj 1024 -> 512


def flops_per_text(cfg: TextConfig, tokens: int = 40) -> float:
    """2 M N K of the layer GEMMs plus 4 T^2 d of attention over all layers, and text_proj on [CLS]: 1.9e10 at 40 tokens."""
    t, d, m = tokens, cfg.hidden, cfg.mlp
    per_layer = 2 * t * d * (3 * d) + 2 * t * d * d + 2 * 2 * t * d * m + 4 * t * t * d
    return float(per_layer * cfg.layers + 2 * d * cfg.embed_dim)


def random_weights(cfg: TextConfig, seed: int) -> dict[str, np.ndarray]:
    """The text tower's seeded weights (cosmos_curate_b200.models.internvideo2.seeded_text_weights) for this config."""
    from cosmos_curate_b200.models.internvideo2 import seeded_text_weights

    return seeded_text_weights(cfg.to_dict(), seed)


def forward(cfg: TextConfig, w: dict, ids, lengths, dtype=torch.float32, device="cpu") -> torch.Tensor:
    """ids int [n][L] ([CLS] ... [SEP] then [PAD]), lengths [n] -> unit-norm embeddings [n][embed_dim] (float32)."""
    W = {k: torch.as_tensor(v).to(device=device, dtype=dtype) for k, v in w.items()}
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    lengths = torch.as_tensor(np.asarray(lengths), dtype=torch.long, device=device)
    n, L = ids.shape
    d, h = cfg.hidden, cfg.heads
    hd = d // h
    ln = lambda x, p: F.layer_norm(x, (d,), W[p + "_w"], W[p + "_b"], cfg.ln_eps)  # noqa: E731
    x = ln((W["tok_emb"][ids] + W["type_emb"]) + W["pos_emb"][:L], "emb_ln")
    keep = (torch.arange(L, device=device)[None, :] < lengths[:, None])[:, None, None, :]  # [n][1][1][L]: keys < length
    for i in range(cfg.layers):
        p = f"L{i}."
        q, k, v = (x @ W[p + "qkv_w"].T + W[p + "qkv_b"]).split(d, dim=-1)
        q, k, v = (a.reshape(n, L, h, hd).transpose(1, 2) for a in (q, k, v))
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=keep, scale=hd**-0.5).transpose(1, 2).reshape(n, L, d)
        x = ln(x + (a @ W[p + "proj_w"].T + W[p + "proj_b"]), p + "ln1")
        y = F.gelu(x @ W[p + "fc1_w"].T + W[p + "fc1_b"]) @ W[p + "fc2_w"].T + W[p + "fc2_b"]
        x = ln(x + y, p + "ln2")
    e = (x[:, 0] @ W["tproj_w"].T + W["tproj_b"]).float()
    return e / e.norm(dim=-1, keepdim=True)
