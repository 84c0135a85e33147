"""Multi-head attention softmax(Q K^T / sqrt(d)) V over a packed fp16 QKV matrix: the float64 reference, the error bound the kernels'
own arithmetic allows, a numpy model of what they round, inputs whose right answer is known bit for bit, and the dispatch rules of
``cb_attention_f16``.

Layout (as the tower writes it): ``qkv`` is ``[n][T][3 * hidden]`` with Q, K, V side by side, ``hidden = heads * head_dim``; the
output is ``[n][T][hidden]``.  The functions take torch tensors on any device (float64 work on the GPU is fine) unless they say
numpy.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

U11 = 2.0**-11  # unit roundoff of fp16 (10 stored mantissa bits)
U24 = 2.0**-24  # unit roundoff of fp32, and the spacing of fp16 subnormals
SELECT_BITS = 11  # selection inputs carry the key index in binary on this many channels: T <= 2048
SELECT_MAG = 10.0  # ... as +-10: the logit gap to any other key is >= 2 * 10^2 / sqrt(head_dim), >= 22 nats at head_dim 80


def split_heads(qkv: torch.Tensor, heads: int):
    """[n][T][3 * hidden] -> q, k, v, each [n][heads][T][head_dim]."""
    n, t, three_hidden = qkv.shape
    hd = three_hidden // 3 // heads
    q, k, v = qkv.view(n, t, 3, heads, hd).permute(2, 0, 3, 1, 4)
    return q, k, v


def merge_heads(o: torch.Tensor) -> torch.Tensor:
    """[n][heads][T][head_dim] -> [n][T][hidden]."""
    n, h, t, hd = o.shape
    return o.permute(0, 2, 1, 3).reshape(n, t, h * hd)


def reference(qkv: torch.Tensor, heads: int):
    """softmax(Q K^T / sqrt(d)) V in float64 from the fp16 inputs, and S_abs = sum_j p_j |v_j| per output element; both [n][T][hidden]."""
    q, k, v = (x.double() for x in split_heads(qkv, heads))
    s = q @ k.transpose(-1, -2) / math.sqrt(q.shape[-1])
    p = torch.softmax(s, dim=-1)
    return merge_heads(p @ v), merge_heads(p @ v.abs())


def bound(ref: torch.Tensor, s_abs: torch.Tensor, qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """Per-element |kernel - reference| that the kernels' arithmetic allows, [n][T][hidden].

    Both kernels compute the scores in fp32 (tensor-core or fma accumulation), p = ex2.approx(fma(s, log2e / sqrt(d), -max)), round p
    to fp16 for the P.V product, sum the unrounded p in fp32, accumulate P.V in fp32, scale by 1 / rowsum and round to fp16.  Terms:

    * output rounding to fp16: 2^-11 |ref|;
    * p rounded to fp16 while the row sum keeps the unrounded p: every term p_j v_j moves by <= 2^-11 p_j |v_j|, so 2^-11 S_abs;
    * fp32 accumulation of P.V over T keys, of the row sum, and the normalisation: (T + 2) 2^-24 (S_abs + |ref|);
    * score error: the fp32 dot products over head_dim (tensor cores may truncate: 2^-23 per add) move every logit by at most
      d 2^-23 max_j sum_i |q_i k_ji| / sqrt(d); the row maximum moves too, and ex2.approx adds 2^-21 relative.  A relative error e_j
      in p_j moves the output by sum_j p_j e_j (v_j - o), so this term is (2 d 2^-23 max_j sum_i |q_i k_ji| / sqrt(d) + 2^-21)
      (S_abs + |ref|);
    * subnormal p (spacing 2^-24, half of it per key) and the fp32 rounding of the ex2 argument (2^-24 |x| relative in p, and
      p |x| ln 2 <= 0.54 for p = 2^-x): 2^-24 T max|v| over the row sum, which is >= 1;
    * the fp16 subnormal floor of the output: 2^-25.
    """
    q, k, v = split_heads(qkv, heads)
    n, h, t, hd = q.shape
    qa, ka = q.double().abs(), k.double().abs()
    dot_abs = (qa @ ka.transpose(-1, -2)).amax(dim=-1, keepdim=True)  # [n][h][T][1]: max_j sum_i |q_i k_ji|
    e_score = merge_heads((2 * hd * 2.0**-23 * dot_abs / math.sqrt(hd) + 2.0**-21).expand(n, h, t, hd))
    vmax = merge_heads(v.double().abs().amax(dim=(-2, -1), keepdim=True).expand(n, h, t, hd))  # per (image, head)
    a, s = ref.abs(), s_abs
    return U11 * a + U11 * s + ((t + 2) * U24 + e_score) * (s + a) + U24 * t * vmax + 2.0**-25


def emulate(qkv: np.ndarray, heads: int) -> np.ndarray:
    """numpy model of what both kernels round: fp32 scores, p = exp2(fma(s, log2e / sqrt(d), -max * log2e / sqrt(d))) in fp32, P
    rounded to fp16 for P.V, fp32 row sums of the unrounded p, output rounded to fp16.  [n][T][3 * hidden] fp16 -> [n][T][hidden] fp16."""
    x = np.asarray(qkv, dtype=np.float16)
    n, t, three_hidden = x.shape
    hd = three_hidden // 3 // heads
    q, k, v = x.astype(np.float32).reshape(n, t, 3, heads, hd).transpose(2, 0, 3, 1, 4)
    c = np.float32(1.4426950408889634) / np.sqrt(np.float32(hd))  # as the host computes scale_log2e
    s = np.matmul(q, k.transpose(0, 1, 3, 2))  # fp32
    mb = s.max(axis=-1, keepdims=True) * c  # fp32 product
    arg = (s.astype(np.float64) * np.float64(c) - mb.astype(np.float64)).astype(np.float32)  # fma: one rounding
    p = np.exp2(arg.astype(np.float64)).astype(np.float32)
    rowsum = p.sum(axis=-1, keepdims=True, dtype=np.float32)
    o = np.matmul(p.astype(np.float16).astype(np.float64), v.astype(np.float64)).astype(np.float32)
    o = (o * (np.float32(1.0) / rowsum)).astype(np.float16)
    return o.transpose(0, 2, 1, 3).reshape(n, t, heads * hd)


# ------------------------------------------------------------------------------------------- structured inputs, exact answers
def key_code(idx: torch.Tensor) -> torch.Tensor:
    """+-SELECT_MAG binary code of each index on SELECT_BITS channels: [...] int -> [..., SELECT_BITS] float32."""
    bits = (idx.long()[..., None] >> torch.arange(SELECT_BITS, device=idx.device)) & 1
    return (bits.float() * 2 - 1) * SELECT_MAG


def boundary_tokens(t: int) -> list[int]:
    """Token indices where the kernels change tile, chunk or path: 16-row tiles, 32-key chunks, the 128-row warpgroup split, the
    256-key tile and the last token."""
    return sorted({i for i in (0, 15, 16, 31, 32, 127, 128, 255, 256, t - 1) if 0 <= i < t})


def selection_inputs(n: int, t: int, heads: int, head_dim: int, seed: int):
    """QKV whose softmax is exactly one-hot after fp16 rounding of P: key j carries the code of j, query i the code of key pi(i).
    Returns (qkv fp16 [n][T][3 * hidden] on the CPU, pi [n][heads][T] int64).  The output row i of (image, head) is V[pi(i)] bit
    for bit.  pi differs per image and head, maps the boundary query rows onto the boundary keys (rotated per unit) and every other
    row onto a random key."""
    assert t <= 2**SELECT_BITS and head_dim >= SELECT_BITS
    g = torch.Generator().manual_seed(seed)
    bnd = boundary_tokens(t)
    pi = torch.randint(0, t, (n, heads, t), generator=g)
    for u in range(n * heads):
        b, h = divmod(u, heads)
        pi[b, h, bnd] = torch.tensor([bnd[(i + u) % len(bnd)] for i in range(len(bnd))])
    q = torch.zeros(n, heads, t, head_dim)
    k = torch.randn(n, heads, t, head_dim, generator=g)  # channels past the code meet zeros in Q: any finite value
    k[..., :SELECT_BITS] = key_code(torch.arange(t)).expand(n, heads, t, SELECT_BITS)
    q[..., :SELECT_BITS] = key_code(pi)
    v = torch.randn(n, heads, t, head_dim, generator=g) * 2
    return pack(q, k, v), pi


def uniform_inputs(n: int, t: int, heads: int, head_dim: int, seed: int):
    """Q = 0, K random, V constant over the tokens of each (image, head, dim) with a different constant per image: p = 1 exactly, the
    row sum is T and sum_j c = T c is exact in fp32, so the output is the constant bit for bit.  Returns (qkv, c [n][heads][head_dim])."""
    g = torch.Generator().manual_seed(seed)
    c = (torch.randn(n, heads, head_dim, generator=g) * 3).half().float()
    q = torch.zeros(n, heads, t, head_dim)
    k = torch.randn(n, heads, t, head_dim, generator=g) * 2
    v = c[:, :, None, :].expand(n, heads, t, head_dim)
    return pack(q, k, v), c


def random_inputs(n: int, t: int, heads: int, head_dim: int, seed: int, kind: str = "normal") -> torch.Tensor:
    """Random QKV (fp16, CPU) of one of these kinds:
    ``normal``: N(0, 1.5^2), as in the tower;  ``sharp``: plus one dominant shared channel in Q and K (rows near one-hot);
    ``large``: logits of magnitude ~10^3 with O(1) differences between keys;  ``ties``: keys repeated in runs of 3 (exactly equal
    logits) with distinct values."""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(n, heads, t, head_dim, generator=g) * 1.5 for _ in range(3))
    if kind == "sharp":
        q[..., 5] += 6.0
        k[..., 5] += 6.0 * torch.rand(n, heads, t, generator=g)
    elif kind == "large":
        big = 32.0 * math.sqrt(head_dim)  # q_0 k_0 ~ 1000 sqrt(d): logits ~ 10^3
        q[..., 0] = big
        k[..., 0] = 32.0 + 0.02 * torch.randn(n, heads, t, generator=g)
        q[..., 1:] *= 0.1
    elif kind == "ties":
        k = k[:, :, torch.arange(t) // 3 * 3]
    else:
        assert kind == "normal", kind
    return pack(q, k, v)


def pack(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """q, k, v [n][heads][T][head_dim] -> fp16 qkv [n][T][3 * hidden]."""
    return torch.cat([merge_heads(x.half()) for x in (q, k, v)], dim=-1).contiguous()


# ------------------------------------------------------------------------------------------------------------ dispatch rules
RESIDENT_SMEM = 100 * 1024  # the mma.sync kernel keeps K and V resident while 2 * t_pad * (HD + 8) halves fit: two CTAs per SM


@dataclass(frozen=True)
class AttnPath:
    name: str
    kernel: str
    head_dims: tuple[int, ...]
    tokens: tuple[int, int]  # inclusive token range this path serves for those head_dims


def _max_resident(hd_pad: int) -> int:
    return RESIDENT_SMEM // (2 * (hd_pad + 8) * 2) // 16 * 16  # largest t_pad whose K and V fit


MAX_T = 2048  # the longest sequence the tests use (the selection code has 11 bits)
# the shapes the tests sweep: every tile, chunk and path boundary of the token count; 560 ends on a 48-key block (a full 32-key
# chunk and a 16-key tail after two streamed 256-key blocks)
SWEEP_T = [1, 2, 15, 16, 17, 31, 32, 33, 48, 127, 128, 129, 130, 191, 192, 193, 255, 256, 257, 258, 288, 289, 352, 353, 560, 729, 1030]
SWEEP_HD = [16, 24, 32, 40, 48, 56, 64, 72, 80]
PATHS = [
    AttnPath("wgmma", "attention_wgmma_kernel<false>", (64,), (129, 255)),
    AttnPath("wgmma_full", "attention_wgmma_kernel<true>", (64,), (256, 257)),
    AttnPath("mma64_resident", "attention_kernel<64, false>", (16, 24, 32, 40, 48, 56, 64), (1, _max_resident(64))),  # 352
    AttnPath("mma64_stream", "attention_kernel<64, true>", (16, 24, 32, 40, 48, 56, 64), (_max_resident(64) + 1, MAX_T)),
    AttnPath("mma80_resident", "attention_kernel<80, false>", (72, 80), (1, _max_resident(80))),  # 288
    AttnPath("mma80_stream", "attention_kernel<80, true>", (72, 80), (_max_resident(80) + 1, MAX_T)),
]


def path_of(t: int, head_dim: int, force_mma: bool = False) -> str | None:
    """The kernel cb_attention_f16 runs for this shape (``CB_ATTN_KERNEL=mma`` is ``force_mma``); None: CB_ERR_UNSUPPORTED."""
    if not force_mma and head_dim == 64 and 129 <= t <= 257:
        return "wgmma_full" if t >= 256 else "wgmma"
    if t <= 0 or head_dim % 8 or head_dim > 80 or head_dim < 16:
        return None
    hd_pad = 64 if head_dim <= 64 else 80
    t_pad = (t + 15) // 16 * 16
    resident = 2 * t_pad * (hd_pad + 8) * 2 <= RESIDENT_SMEM
    return f"mma{hd_pad}_{'resident' if resident else 'stream'}"


def table_path(t: int, head_dim: int, force_mma: bool = False) -> str | None:
    """path_of read from PATHS instead of restating the rules: the CPU tests check that the two agree."""
    for p in PATHS:
        if force_mma and p.name.startswith("wgmma"):
            continue
        if head_dim in p.head_dims and p.tokens[0] <= t <= p.tokens[1]:
            return p.name
    return None
