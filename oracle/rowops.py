"""Oracle for the tower's row kernels (csrc/vit_kernels.cu): LayerNorm, LayerNorm-post, RMSNorm, qk-RMSNorm, token assembly, the CLIP
tail, the SigLIP MAP pool, InternVideo2's clip pool, token mean, tube patches, L2 normalise/score and the affine score.

Every kernel has two models here:

* a float64 reference of the operation (`*_ref`), what the kernel approximates;
* a float32 model (`*_f32`) that rounds exactly as the kernel does: the same summation order (each lane sums its strided float4 as
  (x + y) + (z + w); `warp_sum` is the xor butterfly 16, 8, 4, 2, 1, so every lane ends with the same value; block sums go through
  red[] across the 8 warps of a 256-thread CTA; the pools take per-thread strided max and sum, sum the warps in order, then add the
  slice partials in order; token_mean sums its tokens in order) and the same contraction nvcc emits for sm_90a with the library's
  flags (no fast-math, -fmad on), read from `cuobjdump -sass` of the built library:
    - LayerNorm / RMSNorm squares: a*a + b*b is FMUL(b, b) then FFMA(a, a, .), so `fma(a, a, b * b)`; the pair sums are FADDs;
    - LayerNorm output: FADD(x, -mean), FMUL(., rstd), FFMA(., gamma, beta); RMSNorm output: (x * r) * w, two FMULs;
    - `/ (float)d`, `1.f / x` and `sqrtf` are the IEEE operations (MUFU.RCP / MUFU.RSQ plus the FCHK slow path): correctly rounded;
    - `rsqrtf` is MUFU.RSQ, within 2 ulp (CUDA Math API) - the models take rstd as an argument (see `rstd_candidates`);
    - clip_tail: `q += c * c` and `sc += e * w` are FFMAs; the projection's a.x*p0 + a.y*p1 + a.z*p2 + a.w*p3 is
      FFMA(a.w, p3, FFMA(a.z, p2, FFMA(a.x, p0, a.y * p1))) added to the lane's running sum with an FADD;
    - affine_score: `acc += e * w` is an FFMA; l2norm_score and the pools spell out their fmaf calls (the pools evaluate the d + 1 term
      of their dot product before the d term);
    - `__expf` (pools) is one MUFU.EX2 of x * log2(e): not modelled bit for bit, see `pool_bound`.

Exactness classes (what the GPU tests assert):
  bit-exact:                 l2norm_score, affine_score, token_mean, tube_patches, SigLIP and InternVideo2 assemble;
  bit-exact up to one rsqrtf per row: LayerNorm (every instantiation), LayerNorm-post, RMSNorm, qk-RMSNorm, CLIP assemble, clip_tail -
                             ONE of the <= 5 fp32 candidates around the correctly rounded rsqrt must reproduce the whole row (for
                             clip_tail: emb, feat and score together);
  bounded:                   map_pool and clip_pool on general inputs (`pool_bound`); bit-exact on the uniform and one-hot inputs of
                             `pool_uniform_inputs` / `pool_onehot_inputs`.
"""

from __future__ import annotations

import re
from dataclasses import dataclass
from pathlib import Path

import numpy as np

VIT_KERNELS_CU = Path(__file__).resolve().parent.parent / "cosmos_curate_b200" / "csrc" / "vit_kernels.cu"
F32, F16 = np.float32, np.float16
LN_MAX_D = 1536  # 128 * kLnMaxChunks
RSQRT_ULP = 2  # CUDA Math API: rsqrtf max error 2 ulp

# ------------------------------------------------------------------------------------------------ dispatch (which instantiation runs)
# d >> 7 -> instantiation; every other multiple of 128 up to 1536 runs the generic <0, ...> one.
DISPATCH = {
    "layernorm": ({6: "layernorm_kernel<6,4>", 8: "layernorm_kernel<8,3>", 9: "layernorm_kernel<9,3>"}, "layernorm_kernel<0,3>"),
    "layernorm_post": ({8: "layernorm_post_kernel<8,3>"}, "layernorm_post_kernel<0,3>"),
    "rmsnorm": ({11: "rmsnorm_kernel<11>"}, "rmsnorm_kernel<0>"),
    "qk_rmsnorm": ({11: "qk_rmsnorm_kernel<11>"}, "qk_rmsnorm_kernel<0>"),
}
NORMS = tuple(DISPATCH)
WIDTHS = tuple(128 * k for k in range(1, 13))


def instantiation(kernel: str, d: int) -> str:
    special, generic = DISPATCH[kernel]
    return special.get(d >> 7, generic)


def dispatch_from_source(text: str | None = None) -> dict:
    """DISPATCH as vit_kernels.cu writes it: the `case k:` lines of layernorm_f16's switch and the `d >> 7 == k` tests of the others."""
    text = VIT_KERNELS_CU.read_text() if text is None else text
    out = {}
    for kernel, kname in (("layernorm", "layernorm_kernel"), ("layernorm_post", "layernorm_post_kernel"), ("rmsnorm", "rmsnorm_kernel"),
                          ("qk_rmsnorm", "qk_rmsnorm_kernel")):  # fmt: skip
        body = re.search(rf"\nint {kernel}_f16\(.*?\n}}\n", text, re.S)
        assert body, f"vit_kernels.cu has no host function {kernel}_f16"
        b = body.group(0)
        special = {int(k): f"{kname}<{a.replace(' ', '')}>" for k, a in re.findall(rf"case (\d+): {kname}<([\d, ]+)>", b)}
        m = re.search(rf"if \(d >> 7 == (\d+)\)[^\n]*\n\s*{kname}<([\d, ]+)>", b)
        if m:
            special[int(m.group(1))] = f"{kname}<{m.group(2).replace(' ', '')}>"
        generic = re.findall(rf"(?:default: |else\n\s*){kname}<([\d, ]+)>", b)
        assert len(generic) == 1, f"{kernel}_f16: expected one generic launch, found {generic}"
        out[kernel] = (special, f"{kname}<{generic[0].replace(' ', '')}>")
    return out


# ------------------------------------------------------------------------------------------------ sweep
TOKENS = (1, 2, 255, 256, 257, 729, 1025, 2049)
HEAD_DIMS = (64, 72, 88, 128)  # slices 4, 3, 2, 2: 256, 216, 176, 256 threads busy
POOL_TOWER_HEAD_DIM = {"map": 72, "clip": 88}  # SigLIP So400m's heads, InternVideo2-1B's: every token count runs at these
POOL_BIG_TOKENS = 12289  # (12289 + 256) floats = 50180 bytes: past the 48 KB default, so the call opts in


def pool_sweep(kind: str) -> list[tuple[int, int]]:
    """(head_dim, tokens) for map_pool ("map") or clip_pool ("clip"): every token count at the tower's head_dim, tokens 1, 257 and 2049
    (one warp's worth, one past a CTA's 256 threads, the longest) at every other head_dim, and POOL_BIG_TOKENS (past the 48 KB
    shared-memory default) at 64 and 88."""
    hd0 = POOL_TOWER_HEAD_DIM[kind]
    pts = [(hd0, t) for t in TOKENS] + [(hd, t) for hd in HEAD_DIMS if hd != hd0 for t in (1, 257, 2049)]
    return pts + [(hd, POOL_BIG_TOKENS) for hd in (64, 88)]


def rows_classes(sm: int) -> tuple[int, ...]:
    """1, 7, 8, 9 and 8 sm -+ 1: each CTA handles 8 rows, so these are one partial CTA, one full one, one past it and a grid one CTA
    short of / past one wave of the SMs."""
    return (1, 7, 8, 9, 8 * sm - 1, 8 * sm + 1)


@dataclass(frozen=True)
class NormPoint:
    kernel: str
    d: int
    rows: int

    @property
    def inst(self) -> str:
        return instantiation(self.kernel, self.d)

    @property
    def name(self) -> str:
        return f"{self.kernel}-d{self.d}-r{self.rows}"


def norm_sweep(kernel: str, sm: int) -> list[NormPoint]:
    """Every d = 128 k (k = 1..12); every row class at each specialised width, one row class (in turn) at every width the generic
    instantiation runs, which puts it on every row class too."""
    rc = rows_classes(sm)
    special = DISPATCH[kernel][0]
    pts = []
    for k, d in enumerate(WIDTHS):
        if (d >> 7) in special:
            pts += [NormPoint(kernel, d, r) for r in rc]
        else:
            pts.append(NormPoint(kernel, d, rc[k % len(rc)]))
    return pts


# ------------------------------------------------------------------------------------------------ float32 arithmetic
def fma(a, b, c) -> np.ndarray:
    """Correctly rounded float32 fma(a, b, c): the float64 product is exact, the float64 sum is made round-to-odd (two spare bits are
    enough for the second rounding to float32 to be correct)."""
    a, b, c = (np.asarray(t, dtype=np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)  # TwoSum: s + err == p + c exactly
    bits = s.view(np.int64) if s.ndim else np.asarray(s).reshape(1).view(np.int64)
    even = (bits & 1) == 0
    fix = (err != 0) & even.reshape(s.shape) & np.isfinite(s)
    if np.any(fix):
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def warp_sum(v: np.ndarray) -> np.ndarray:
    """v float32 [..., 32] -> the xor-butterfly sum every lane ends with, [...]."""
    v = v.astype(F32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., np.arange(32) ^ o]
    return v[..., 0]


def block_sum(v: np.ndarray) -> np.ndarray:
    """v float32 [..., 256] (one value per thread) -> clip_tail's block_sum: warp sums into red[0..7], then warp 0 sums red[] with
    lanes 8..31 reading zero."""
    w = warp_sum(v.reshape(*v.shape[:-1], 8, 32))
    return warp_sum(np.concatenate([w, np.zeros((*w.shape[:-1], 24), F32)], axis=-1))


def rsqrt_rn(x) -> np.ndarray:
    """Correctly rounded float32 1/sqrt(x)."""
    return (1.0 / np.sqrt(np.asarray(x, dtype=np.float64))).astype(F32)


def ulp_step(x: np.ndarray, k: int) -> np.ndarray:
    """x moved k float32 ulps (positive x)."""
    out = np.asarray(x, dtype=F32).copy()
    for _ in range(abs(k)):
        out = np.nextafter(out, F32(np.inf) if k > 0 else F32(0))
    return out


def rstd_candidates(arg) -> list[tuple[int, np.ndarray]]:
    """The fp32 values rsqrtf(arg) may return: the correctly rounded one and RSQRT_ULP ulps either side, as (offset, value)."""
    r = rsqrt_rn(arg)
    return [(k, ulp_step(r, k)) for k in range(-RSQRT_ULP, RSQRT_ULP + 1)]


def lanes(x: np.ndarray) -> np.ndarray:
    """Rows [R][d] as the warp reads them: [R][chunk][lane][4], element ((chunk * 32) + lane) * 4 + j."""
    r, d = x.shape
    return x.reshape(r, d // 128, 32, 4)


# ------------------------------------------------------------------------------------------------ LayerNorm family
def ln_stats(x: np.ndarray, eps: float, variant: str = "kernel") -> tuple[np.ndarray, np.ndarray]:
    """ln_row's statistics: (mean [R], the rsqrtf argument var + eps [R]).  `variant` restates a wrong formula for the tests that show
    the acceptance rule rejects it: "unbiased", "eps_outside" (returns var; the caller adds eps after the root), "one_pass"."""
    x = x.astype(F32)
    r, d = x.shape
    v = lanes(x)
    s = np.zeros((r, 32), F32)
    for i in range(v.shape[1]):
        s = s + ((v[:, i, :, 0] + v[:, i, :, 1]) + (v[:, i, :, 2] + v[:, i, :, 3]))
    mean = warp_sum(s) / F32(d)
    q = np.zeros((r, 32), F32)
    if variant == "one_pass":
        for i in range(v.shape[1]):
            a, b, c, e = (v[:, i, :, j] for j in range(4))
            q = q + (fma(a, a, b * b) + fma(c, c, e * e))
        var = warp_sum(q) / F32(d) - mean * mean
        return mean, (var + F32(eps)).astype(F32)
    c4 = v - mean[:, None, None, None]
    for i in range(v.shape[1]):
        a, b, c, e = (c4[:, i, :, j] for j in range(4))
        q = q + (fma(a, a, b * b) + fma(c, c, e * e))
    div = F32(d - 1) if variant == "unbiased" else F32(d)
    var = warp_sum(q) / div
    return mean, (var if variant == "eps_outside" else var + F32(eps)).astype(F32)


def ln_apply(x: np.ndarray, mean: np.ndarray, rstd: np.ndarray, gamma: np.ndarray, beta: np.ndarray) -> np.ndarray:
    """fma((x - mean) * rstd, gamma, beta), float32 [R][d]."""
    return fma((x.astype(F32) - mean[:, None]) * rstd[:, None], gamma[None, :], beta[None, :])


def layernorm_ref(x, gamma, beta, eps) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    mu = x.mean(1, keepdims=True)
    var = ((x - mu) ** 2).mean(1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64)


def rms_stats(x: np.ndarray, eps: float, variant: str = "kernel") -> np.ndarray:
    """rmsnorm_kernel's rsqrtf argument mean(x^2) + eps [R]; variant "centred" subtracts the mean first (a LayerNorm, wrong here)."""
    x = x.astype(F32)
    if variant == "centred":
        x = x - (x.astype(np.float64).mean(1, keepdims=True)).astype(F32)
    r, d = x.shape
    v = lanes(x)
    s = np.zeros((r, 32), F32)
    for i in range(v.shape[1]):
        a, b, c, e = (v[:, i, :, j] for j in range(4))
        s = s + (fma(a, a, b * b) + fma(c, c, e * e))
    return (warp_sum(s) / F32(d) + F32(eps)).astype(F32)


def rms_apply(x: np.ndarray, r: np.ndarray, w: np.ndarray) -> np.ndarray:
    return (x.astype(F32) * r[:, None]) * w[None, :].astype(F32)


def rmsnorm_ref(x, w, eps) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    return x / np.sqrt((x * x).mean(1, keepdims=True) + eps) * np.asarray(w, np.float64)


def match_rows(got: np.ndarray, stats_arg: np.ndarray, apply) -> tuple[np.ndarray, np.ndarray]:
    """The acceptance rule of the rsqrtf class.  got: the kernel's rows [R][...] (any dtype, compared bitwise); apply(rstd [R]) -> the
    model's rows for that rstd, same dtype and shape.  Returns (offset [R] of the first candidate, nearest the correctly rounded
    value first, that reproduces the WHOLE row bit for bit, or a sentinel 99 when none does; the mismatch count of the best candidate)."""
    order = sorted(rstd_candidates(stats_arg), key=lambda kv: (abs(kv[0]), kv[0]))
    off = np.full(got.shape[0], 99, np.int64)
    best = np.full(got.shape[0], np.iinfo(np.int64).max, np.int64)
    gb = _bits(got).reshape(got.shape[0], -1)
    for k, r in order:
        want = _bits(apply(r)).reshape(got.shape[0], -1)
        bad = (want != gb).sum(1)
        best = np.minimum(best, bad)
        off = np.where((off == 99) & (bad == 0), k, off)
    return off, best


def _bits(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a)
    return a.view({2: np.int16, 4: np.int32, 8: np.int64}[a.dtype.itemsize])


# ------------------------------------------------------------------------------------------------ token assembly
def assemble_f32(patch, cls, pos, gamma, beta, rstd, eps, n: int, tokens: int, grid2: int, pos_shift: int = 0) -> tuple:
    """assemble_kernel: rows [n * tokens][d] before the norm (the summed inputs) and, for CLIP, (mean, arg) of each row.  The caller
    applies ln_apply with the chosen rstd; SigLIP (gamma None) returns the sums themselves.  pos_shift = -1 restates the wrong
    "pos[t - 1]"."""
    d = pos.shape[1]
    has_cls = tokens != grid2
    src = np.empty((n, tokens, d), F32)
    p = patch.reshape(n, grid2, d)
    if has_cls:
        src[:, 0] = cls
        src[:, 1:] = p
    else:
        src[:] = p
    t = np.clip(np.arange(tokens) + pos_shift, 0, tokens - 1)
    summed = (src + pos[t][None]).reshape(n * tokens, d).astype(F32)
    if gamma is None:
        return summed, None
    return summed, ln_stats(summed, eps)


# ------------------------------------------------------------------------------------------------ CLIP tail
def clip_tail_stats(x: np.ndarray, eps: float) -> tuple[np.ndarray, np.ndarray]:
    """clip_tail_kernel's post-LN statistics on rows x [n][d]: (mean, var + eps), threads striding by 256."""
    n, d = x.shape
    x = x.astype(F32)
    pad = (-d) % 256
    xp = np.concatenate([x, np.zeros((n, pad), F32)], 1).reshape(n, -1, 256)
    s = np.zeros((n, 256), F32)
    for j in range(xp.shape[1]):
        s = s + xp[:, j]
    mean = block_sum(s) / F32(d)
    c = np.concatenate([x - mean[:, None], np.zeros((n, pad), F32)], 1).reshape(n, -1, 256)
    q = np.zeros((n, 256), F32)
    for j in range(c.shape[1]):
        q = fma(c[:, j], c[:, j], q)
    return mean, (block_sum(q) / F32(d) + F32(eps)).astype(F32)


def _strided_fma_dot(a: np.ndarray, b: np.ndarray, threads: int) -> np.ndarray:
    """Per-thread running fma(a[i], b[i], acc) over i = tid, tid + threads, ...: [n][threads]."""
    n, m = a.shape
    pad = (-m) % threads
    ap = np.concatenate([a, np.zeros((n, pad), F32)], 1).reshape(n, -1, threads)
    bp = np.concatenate([b, np.zeros((n, pad), F32)], 1).reshape(n, -1, threads)
    acc = np.zeros((n, threads), F32)
    for j in range(ap.shape[1]):
        acc = fma(ap[:, j], bp[:, j], acc)
    return acc


def clip_tail_f32(x, mean, rstd, gamma, beta, proj, aes_w, aes_b) -> tuple[np.ndarray, np.ndarray, np.ndarray | None]:
    """(emb, feat, score) of clip_tail_kernel for rows x [n][d] with the given rstd [n]."""
    n, d = x.shape
    pooled = ln_apply(x, mean, rstd, gamma, beta)
    if proj is not None:
        pv = lanes(pooled)[:, None]  # lane l reads pooled[i .. i + 3], i = 4 l + 128 j: [n][1][chunk][lane][4]
        wv = proj.astype(F32).reshape(1, proj.shape[0], d // 128, 32, 4)  # [1][out][chunk][lane][4]
        acc = np.zeros((n, proj.shape[0], 32), F32)
        for j in range(d // 128):
            a, p = wv[:, :, j], pv[:, :, j]
            acc = acc + fma(a[..., 3], p[..., 3], fma(a[..., 2], p[..., 2], fma(a[..., 0], p[..., 0], a[..., 1] * p[..., 1])))
        feat = warp_sum(acc)
    else:
        feat = pooled
    n2 = block_sum(_strided_fma_dot(feat, feat, 256))
    inv = F32(1) / np.sqrt(n2)
    emb = feat * inv[:, None]
    score = None
    if aes_w is not None:
        sc = _strided_fma_dot(emb, np.broadcast_to(aes_w.astype(F32), emb.shape), 256)
        score = block_sum(sc) + F32(aes_b)
    return emb, feat, score


def clip_tail_ref(x, gamma, beta, eps, proj, aes_w, aes_b):
    pooled = layernorm_ref(x, gamma, beta, eps)
    feat = pooled @ np.asarray(proj, np.float64).T if proj is not None else pooled
    emb = feat / np.linalg.norm(feat, axis=1, keepdims=True)
    score = emb @ np.asarray(aes_w, np.float64) + aes_b if aes_w is not None else None
    return emb, feat, score


# ------------------------------------------------------------------------------------------------ L2 / scores / mean / patches
def l2norm_score_f32(feat: np.ndarray, aes_w, aes_b) -> tuple[np.ndarray, np.ndarray | None]:
    """l2norm_score_kernel: one warp per row, lanes striding by 32."""
    feat = feat.astype(F32)
    n2 = warp_sum(_strided_fma_dot(feat, feat, 32))
    inv = F32(1) / np.sqrt(n2)
    emb = feat * inv[:, None]
    score = None
    if aes_w is not None:
        score = warp_sum(_strided_fma_dot(emb, np.broadcast_to(aes_w.astype(F32), emb.shape), 32)) + F32(aes_b)
    return emb, score


def affine_score_f32(emb: np.ndarray, w: np.ndarray, b: float) -> np.ndarray:
    return warp_sum(_strided_fma_dot(emb.astype(F32), np.broadcast_to(w.astype(F32), emb.shape), 32)) + F32(b)


def token_mean_f32(h: np.ndarray, divisor_shift: int = 0) -> np.ndarray:
    """h [n][T][d] -> tokens summed in order, / T (divisor_shift = -1 restates the wrong T - 1)."""
    s = np.zeros((h.shape[0], h.shape[2]), F32)
    for t in range(h.shape[1]):
        s = s + h[:, t].astype(F32)
    return s / F32(h.shape[1] + divisor_shift)


def tube_patches_f32(tubes: np.ndarray, patch: int, k_pad: int, order: str = "cyx") -> np.ndarray:
    """tubes [F][3][S][S] -> fp16 [F][(S/P)^2][k_pad], k = (c, y, x) ("cxy": y and x transposed; "yxc": channel last - both wrong)."""
    f, _, s, _ = tubes.shape
    g = s // patch
    t = tubes[:, :, : g * patch, : g * patch].reshape(f, 3, g, patch, g, patch)  # f c gy y gx x
    perm = {"cyx": (0, 2, 4, 1, 3, 5), "cxy": (0, 2, 4, 1, 5, 3), "yxc": (0, 2, 4, 3, 5, 1)}[order]
    rows = t.transpose(perm).reshape(f, g * g, 3 * patch * patch)
    out = np.zeros((f, g * g, k_pad), F16)
    out[..., : rows.shape[-1]] = rows.astype(F16)
    return out


# ------------------------------------------------------------------------------------------------ pools
def pool_slices(head_dim: int) -> int:
    return max(1, 256 // head_dim)


def pool_scores_f32(k: np.ndarray, qh: np.ndarray) -> np.ndarray:
    """k fp16 [n][T][hd], qh fp32 [n][hd] -> s [n][T]: s = fmaf(k[d], q[d], fmaf(k[d+1], q[d+1], s)) for d = 0, 2, ..."""
    kf = k.astype(F32)
    s = np.zeros(k.shape[:2], F32)
    for d in range(0, k.shape[2], 2):
        s = fma(kf[..., d], qh[:, None, d], fma(kf[..., d + 1], qh[:, None, d + 1], s))
    return s


def pool_f32(k: np.ndarray, v: np.ndarray, qh: np.ndarray, expf=None) -> np.ndarray:
    """One query per (image, head): k, v fp16 [n][T][hd] (one head), qh fp32 [n][hd] as the kernel holds it (map_pool: q; clip_pool:
    q * scale).  expf(x float32) -> float32 stands in for __expf (default: float64 exp rounded, exact for the pool_*_inputs classes)."""
    expf = expf or (lambda x: np.exp(x.astype(np.float64)).astype(F32))
    n, t, hd = k.shape
    s = pool_scores_f32(k, qh)
    mx = s.max(1)
    e = expf(s - mx[:, None])
    pad = (-t) % 256
    ep = np.concatenate([e, np.zeros((n, pad), F32)], 1).reshape(n, -1, 256)
    acc = np.zeros((n, 256), F32)
    for j in range(ep.shape[1]):
        acc = acc + ep[:, j]
    w = warp_sum(acc.reshape(n, 8, 32))
    tot = np.zeros(n, F32)
    for i in range(8):
        tot = tot + w[:, i]
    inv = F32(1) / tot
    sl = pool_slices(hd)
    vf = v.astype(F32)
    outacc = np.zeros((n, hd), F32)
    for j in range(sl):
        part = np.zeros((n, hd), F32)
        for tt in range(j, t, sl):
            part = fma(e[:, tt, None], vf[:, tt], part)
        outacc = outacc + part
    return (outacc * inv[:, None]).astype(F16)


def pool_ref(k, v, qh) -> np.ndarray:
    s = np.einsum("ntd,nd->nt", np.asarray(k, np.float64), np.asarray(qh, np.float64))
    p = np.exp(s - s.max(1, keepdims=True))
    return np.einsum("nt,ntd->nd", p / p.sum(1, keepdims=True), np.asarray(v, np.float64))


def pool_bound(k, v, qh) -> np.ndarray:
    """Per-output bound on |pool - pool_ref| [n][hd].

    With p_t = exp(x_t), x_t = s_t - max s <= 0, the kernel's p'_t = __expf(x'_t) carries
      * the documented __expf error, (2 + floor(|1.173 x|)) ulp, i.e. relative e_t <= (2 + floor(1.173 |x_t|)) 2^-23;
      * the fp32 dot product error of s_t and of max s, |x'_t - x_t| <= 2 g_hd sum_d |k q| (g_m = m 2^-24 / (1 - m 2^-24)), so a
        relative factor exp(2 g_hd max_t sum|kq|) - 1 =: e_s on every p_t.
    o' = sum p'_t v_t / sum p'_t moves from o by at most 2 (E + e_s) max|v| / (1 - E - e_s), E = sum p_t e_t / sum p_t (weighted: the
    keys far below the maximum contribute both large e_t and tiny p_t).  The fp32 sums add g_(T/slices + slices + 2) sum p|v| / sum p
    for the numerator, g_(T/256 + 8 + 8) for the denominator, and the final product and 1 / tot one rounding each (u = 2^-24).
    fp16 rounding of the result adds half an fp16 ulp of |o| + that bound.
    """
    k, v, qh = (np.asarray(a, np.float64) for a in (k, v, qh))
    n, t, hd = k.shape
    u = 2.0**-24
    g = lambda m: m * u / (1 - m * u)  # noqa: E731
    s = np.einsum("ntd,nd->nt", k, qh)
    x = s - s.max(1, keepdims=True)
    p = np.exp(x)
    e_t = (2 + np.floor(1.173 * np.abs(x))) * 2.0**-23
    E = (p * e_t).sum(1) / p.sum(1)
    e_s = np.expm1(2 * g(hd) * np.abs(k * qh[:, None]).sum(2).max(1))
    vmax = np.abs(v).max(1)
    pv = np.einsum("nt,ntd->nd", p, np.abs(v)) / p.sum(1, keepdims=True)
    sl = pool_slices(hd)
    err32 = 2 * (E + e_s)[:, None] * vmax / (1 - E - e_s)[:, None]
    err32 = err32 + (g(t // sl + sl + 2) + g(t // 256 + 16) + 3 * u) * (pv + err32)
    o = np.abs(pool_ref(k, v, qh))
    return err32 + 0.5 * f16_ulp(o + err32)


def f16_ulp(x: np.ndarray) -> np.ndarray:
    x = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0**-14)
    return 2.0 ** (np.floor(np.log2(x)) - 10)


def pool_uniform_inputs(n: int, t: int, hd: int, seed: int):
    """Every key equal, so every score is equal and every __expf(0) is exactly 1; V integers / 8 in [-8, 8], whose sums over <= 2049
    tokens are exact in fp32.  Returns (k, v, q) with k, v fp16 [n][T][hd], q fp32 [n][hd]."""
    r = np.random.default_rng(seed)
    k = np.broadcast_to(r.standard_normal((n, 1, hd)), (n, t, hd)).astype(F16)
    v = (r.integers(-64, 65, (n, t, hd)) / 8).astype(F16)
    q = r.standard_normal((n, hd)).astype(F32)
    return np.ascontiguousarray(k), v, q


def onehot_code(t: np.ndarray, d: np.ndarray) -> np.ndarray:
    """V[t][d] of the one-hot class: fp16-exact and distinct per (t mod 1024, d), so a wrong winner names itself."""
    return ((t * 7 + d * 3) % 1024 / 4 - 128).astype(F16)


def pool_onehot_inputs(n: int, t: int, hd: int, seed: int, scale: float = 1.0):
    """Keys zero except key j(image) = 32 sign(q), whose score leads every other key's (0) by >= 32 hd scale >= 120 nats for the shapes
    used: every other __expf(x) has x <= -120, below fp32's smallest subnormal (2^-149 = e^-103.3) whether or not ex2 flushes, so the
    output is V[j] exactly.  q = +-(1 + U[0, 1)) is the unscaled query; qh = q * scale is what the kernel multiplies with.  Returns
    (k, v, q, j)."""
    r = np.random.default_rng(seed)
    q = (np.where(r.random((n, hd)) < 0.5, -1, 1) * (1 + r.random((n, hd)))).astype(F32)
    j = r.integers(0, t, n)
    k = np.zeros((n, t, hd), F16)
    k[np.arange(n), j] = (32 * np.sign(q)).astype(F16)
    tt, dd = np.meshgrid(np.arange(t), np.arange(hd), indexing="ij")
    v = np.broadcast_to(onehot_code(tt, dd), (n, t, hd)).copy()
    return k, v, q, j
