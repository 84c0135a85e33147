"""Thin Python layer over the C ABI: torch tensors are only zero-copy containers (data_ptr()).

Nothing here computes on the data path; every operation is a call into libcurate_b200.so.
"""

from __future__ import annotations

import ctypes as C
import os
import weakref

import numpy as np
import torch

from . import _lib
from ._lib import Iv2Cfg, Iv2TextCfg, SurfacePool, VitCfg, check

try:
    from loguru import logger
except ImportError:
    import logging

    logger = logging.getLogger(__name__)

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)  # reference: cosmos_curate/models/clip.py:57-60
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
IMAGENET_MEAN = (0.485, 0.456, 0.406)  # reference: cosmos_curate/models/internvideo2_mm.py:378-379
IMAGENET_STD = (0.229, 0.224, 0.225)

_TORCH_DT = {torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16, torch.float32: _lib.DT_F32}


def _f3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


def _stream_ptr(stream=None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


# NV12 -> RGB arithmetic by name: "opencv" (CV-CUDA / cv2.cvtColor semantics, the reference's CUDA branch) or "swscale"
# (libswscale's yuv420p -> rgb24, the reference's CPU decode branch)
COLOURS = {"swscale": _lib.FMT_NV12_SWS, "opencv": _lib.FMT_NV12}


def check_colour(colour: str) -> str:
    """`colour` when it is a key of COLOURS, else ValueError (stages check it at construction, not at the first decode)."""
    if colour not in COLOURS:
        raise ValueError(f"colour={colour!r} not in {tuple(COLOURS)}")
    return colour


def even_size(width: int, height: int) -> tuple[int, int]:
    """Surface size of a width x height stream: 4:2:0 chroma covers 2x2 pixels, so odd sizes round up."""
    return (width + 1) & ~1, (height + 1) & ~1


class _Handle:
    """A library object behind `h`: `_destroy()` runs once, from close() or when the wrapper is collected."""

    h = None

    def _destroy(self) -> None:
        raise NotImplementedError

    def close(self):
        if self.h:
            self._destroy()
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class Context(_Handle):
    """One per process/GPU (cb_init).  Fails loudly when the library or a CUDA device is missing."""

    def __init__(self, device: int | None = None):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.CurateB200Error(-1, "Context", "no CUDA device; this path has no CPU fallback")
        self.device = torch.cuda.current_device() if device is None else int(device)
        torch.cuda.set_device(self.device)
        torch.cuda.init()
        h = C.c_void_p()
        check(self.lib.cb_init(self.device, C.byref(h)), "cb_init")
        self.h = h
        self._children = weakref.WeakSet()  # towers / decoders created on this context: closed before it

    def _destroy(self):
        for child in list(self._children):
            child.close()
        self.lib.cb_destroy(self.h)

    def launch_count(self) -> int:
        return int(self.lib.cb_launch_count(self.h))

    PROF_CATEGORIES = ("preprocess", "gemm", "layernorm", "attention", "other", "conv")

    def profile_begin(self) -> None:
        check(self.lib.cb_profile_begin(self.h), "cb_profile_begin", self.h)

    def profile_end(self) -> dict:
        n = len(self.PROF_CATEGORIES)
        ms, cnt = (C.c_float * n)(), (C.c_int * n)()
        check(self.lib.cb_profile_end(self.h, _stream_ptr(), ms, cnt, n), "cb_profile_end", self.h)
        return {k: {"ms": float(ms[i]), "launches": int(cnt[i])} for i, k in enumerate(self.PROF_CATEGORIES)}

    def device_info(self) -> dict:
        sm, ma, mi, mem = C.c_int(), C.c_int(), C.c_int(), C.c_size_t()
        check(self.lib.cb_device_info(self.h, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(mem)), "cb_device_info", self.h)
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "total_mem": mem.value}

    # ---- surfaces -----------------------------------------------------------------------------
    def nv12_pool(self, buf: torch.Tensor, width: int, height: int, luma_rows: int | None = None, colour: str = "opencv") -> "Pool":
        """buf: uint8 cuda [slots, rows, pitch] with rows >= luma_rows + height/2.  colour: a key of COLOURS."""
        assert buf.is_cuda and buf.dtype == torch.uint8 and buf.dim() == 3 and buf.is_contiguous()
        luma_rows = height if luma_rows is None else luma_rows
        assert buf.shape[1] >= luma_rows + height // 2
        return Pool(buf, SurfacePool(buf.data_ptr(), buf.shape[1] * buf.shape[2], width, height, buf.shape[2], luma_rows, COLOURS[colour]))

    def rgb_pool(self, frames: torch.Tensor) -> "Pool":
        """frames: uint8 cuda [n, H, W, 3] (contiguous).  Rows are re-pitched to a 16-byte multiple if needed."""
        assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3
        n, h, w, _ = frames.shape
        row = 3 * w
        pitch = (row + 15) & ~15
        if pitch != row or not frames.is_contiguous():
            buf = torch.zeros((n, h, pitch), dtype=torch.uint8, device=frames.device)
            buf[:, :, :row] = frames.reshape(n, h, row)
        else:
            buf = frames.reshape(n, h, row)
        stride = h * pitch
        if stride % 16:
            pad = torch.zeros((n, (stride + 15) // 16 * 16), dtype=torch.uint8, device=frames.device)
            pad[:, :stride] = buf.reshape(n, stride)
            buf, stride = pad, pad.shape[1]
        return Pool(buf, SurfacePool(buf.data_ptr(), stride, w, h, pitch, h, _lib.FMT_RGB24))

    # ---- preprocess ---------------------------------------------------------------------------
    def _slots(self, pool: "Pool", slots):
        n_slots = pool.buf.shape[0]
        arr = np.arange(n_slots, dtype=np.int32) if slots is None else np.ascontiguousarray(slots, dtype=np.int32)
        return arr, arr.ctypes.data_as(C.POINTER(C.c_int32))

    def preprocess_clip(self, pool: "Pool", slots=None, res: int = 224, dtype=torch.float16, layout: str = "nchw", patch: int = 0,
                        k_pad: int = 0, mean=CLIP_MEAN, std=CLIP_STD, out: torch.Tensor | None = None) -> torch.Tensor:
        arr, ptr = self._slots(pool, slots)
        n = len(arr)
        if layout == "nchw":
            shape, lay = (n, 3, res, res), _lib.LAYOUT_NCHW
        else:
            g = res // patch
            shape, lay = (n, g * g, k_pad), _lib.LAYOUT_PATCH
        if out is None:
            out = torch.empty(shape, dtype=dtype, device=pool.buf.device)
        check(self.lib.cb_preprocess_clip(self.h, C.byref(pool.desc), ptr, n, res, lay, patch, k_pad, _TORCH_DT[dtype], _f3(mean), _f3(std),
                                          out.data_ptr(), _stream_ptr()), "cb_preprocess_clip", self.h)  # fmt: skip
        return out

    def preprocess_clip_u8(self, pool: "Pool", slots=None, res: int = 224) -> torch.Tensor:
        arr, ptr = self._slots(pool, slots)
        out = torch.empty((len(arr), 3, res, res), dtype=torch.uint8, device=pool.buf.device)
        check(self.lib.cb_preprocess_clip_u8(self.h, C.byref(pool.desc), ptr, len(arr), res, out.data_ptr(), _stream_ptr()),
              "cb_preprocess_clip_u8", self.h)  # fmt: skip
        return out

    def preprocess_bilinear_u8(self, pool: "Pool", out_w: int, out_h: int, slots=None) -> torch.Tensor:
        arr, ptr = self._slots(pool, slots)
        out = torch.empty((len(arr), out_h, out_w, 3), dtype=torch.uint8, device=pool.buf.device)
        check(self.lib.cb_preprocess_bilinear_u8(self.h, C.byref(pool.desc), ptr, len(arr), out_w, out_h, out.data_ptr(), _stream_ptr()),
              "cb_preprocess_bilinear_u8", self.h)  # fmt: skip
        return out

    def resize_cubic_u8(self, pool: "Pool", out_w: int, out_h: int, slots=None, mode: int = _lib.CUBIC_IPP) -> torch.Tensor:
        """cv2.resize(frame, (out_w, out_h), INTER_CUBIC) per frame of the pool -> uint8 cuda [n, out_h, out_w, 3]."""
        arr, ptr = self._slots(pool, slots)
        out = torch.empty((len(arr), out_h, out_w, 3), dtype=torch.uint8, device=pool.buf.device)
        check(self.lib.cb_resize_cubic_u8(self.h, C.byref(pool.desc), ptr, len(arr), out_w, out_h, mode, out.data_ptr(), _stream_ptr()),
              "cb_resize_cubic_u8", self.h)  # fmt: skip
        return out

    def video_tube(self, pool: "Pool", out_w: int, out_h: int, slots=None, mean=IMAGENET_MEAN, std=IMAGENET_STD, want_u8: bool = False):
        """cv2.resize(frame, (out_w, out_h)) + ((x / 255 - mean) / std) per frame -> float32 cuda [n, 3, out_h, out_w]
        (internvideo2_mm.py:385-405); with want_u8 also the resized uint8 [n, out_h, out_w, 3] frames."""
        arr, ptr = self._slots(pool, slots)
        out = torch.empty((len(arr), 3, out_h, out_w), dtype=torch.float32, device=pool.buf.device)
        u8 = torch.empty((len(arr), out_h, out_w, 3), dtype=torch.uint8, device=pool.buf.device) if want_u8 else None
        check(self.lib.cb_video_tube(self.h, C.byref(pool.desc), ptr, len(arr), out_w, out_h, _f3(mean), _f3(std), out.data_ptr(),
                                     u8.data_ptr() if want_u8 else None, _stream_ptr()), "cb_video_tube", self.h)  # fmt: skip
        return (out, u8) if want_u8 else out

    def nv12_to_rgb(self, pool: "Pool", slots=None) -> torch.Tensor:
        arr, ptr = self._slots(pool, slots)
        out = torch.empty((len(arr), pool.desc.height, pool.desc.width, 3), dtype=torch.uint8, device=pool.buf.device)
        check(self.lib.cb_nv12_to_rgb(self.h, C.byref(pool.desc), ptr, len(arr), out.data_ptr(), _stream_ptr()), "cb_nv12_to_rgb", self.h)
        return out

    # ---- building blocks (parity tests) -----------------------------------------------------------
    def gemm(self, a: torch.Tensor, w: torch.Tensor, bias=None, residual=None, epilogue: int = _lib.EPI_NONE, out_f32: bool = False):
        m, k = a.shape
        n = w.shape[0]
        assert a.dtype == torch.float16 and w.dtype == torch.float16 and w.shape[1] == k and a.is_contiguous() and w.is_contiguous()
        if out_f32:
            out = residual if residual is not None else torch.empty((m, n), dtype=torch.float32, device=a.device)
            o32, o16 = out.data_ptr(), None
        else:
            out = torch.empty((m, n), dtype=torch.float16, device=a.device)
            o32, o16 = None, out.data_ptr()
        check(self.lib.cb_gemm_f16(self.h, a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                   residual.data_ptr() if residual is not None else None, o32, o16, m, n, k, epilogue, _stream_ptr()),
              "cb_gemm_f16", self.h)  # fmt: skip
        return out

    def gemm_ex(self, a: torch.Tensor, w: torch.Tensor, bias=None, gamma=None, residual=None, epilogue: int = _lib.EPI_NONE,
                out_f32: bool = False) -> torch.Tensor:
        """cb_gemm_f16_ex: gemm() plus the per-column LayerScale `gamma` (fp32 output)."""
        m, k = a.shape
        n = w.shape[0]
        assert a.dtype == torch.float16 and w.dtype == torch.float16 and w.shape[1] == k and a.is_contiguous() and w.is_contiguous()
        if out_f32:
            out = residual if residual is not None else torch.empty((m, n), dtype=torch.float32, device=a.device)
            o32, o16 = out.data_ptr(), None
        else:
            out = torch.empty((m, n), dtype=torch.float16, device=a.device)
            o32, o16 = None, out.data_ptr()
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        check(self.lib.cb_gemm_f16_ex(self.h, a.data_ptr(), w.data_ptr(), ptr(bias), ptr(gamma), ptr(residual), o32, o16, m, n, k, epilogue,
                                      _stream_ptr()), "cb_gemm_f16_ex", self.h)  # fmt: skip
        return out

    def rmsnorm(self, x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
        rows, d = x.shape
        y = torch.empty((rows, d), dtype=torch.float16, device=x.device)
        check(self.lib.cb_rmsnorm_f16(self.h, x.data_ptr(), weight.data_ptr(), y.data_ptr(), rows, d, eps, _stream_ptr()), "cb_rmsnorm_f16", self.h)
        return y

    def qk_rmsnorm_(self, qkv: torch.Tensor, q_weight: torch.Tensor, k_weight: torch.Tensor, eps: float) -> torch.Tensor:
        """In place on fp16 qkv [rows][3 * d]."""
        rows, three_d = qkv.shape
        check(self.lib.cb_qk_rmsnorm_f16(self.h, qkv.data_ptr(), q_weight.data_ptr(), k_weight.data_ptr(), rows, three_d // 3, eps, _stream_ptr()),
              "cb_qk_rmsnorm_f16", self.h)  # fmt: skip
        return qkv

    def attention_stream(self, qkv: torch.Tensor, heads: int) -> torch.Tensor:
        n, t, three_d = qkv.shape
        d = three_d // 3
        out = torch.empty((n, t, d), dtype=torch.float16, device=qkv.device)
        check(self.lib.cb_attention_stream_f16(self.h, qkv.data_ptr(), out.data_ptr(), n, t, heads, d // heads, _stream_ptr()),
              "cb_attention_stream_f16", self.h)  # fmt: skip
        return out

    def layernorm(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
        rows, d = x.shape
        y = torch.empty((rows, d), dtype=torch.float16, device=x.device)
        check(self.lib.cb_layernorm_f16(self.h, x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), rows, d, eps, _stream_ptr()),
              "cb_layernorm_f16", self.h)  # fmt: skip
        return y

    def attention(self, qkv: torch.Tensor, heads: int) -> torch.Tensor:
        n, t, three_d = qkv.shape
        d = three_d // 3
        out = torch.empty((n, t, d), dtype=torch.float16, device=qkv.device)
        check(self.lib.cb_attention_f16(self.h, qkv.data_ptr(), out.data_ptr(), n, t, heads, d // heads, _stream_ptr()), "cb_attention_f16", self.h)
        return out

    def attention_masked(self, qkv: torch.Tensor, heads: int, lengths: torch.Tensor) -> torch.Tensor:
        """cb_attention_masked_f16: sequence i of qkv [n][T][3 * hidden] attends to its first lengths[i] keys (int32 cuda [n])."""
        n, t, three_d = qkv.shape
        d = three_d // 3
        assert lengths.is_cuda and lengths.dtype == torch.int32 and lengths.shape == (n,)
        out = torch.empty((n, t, d), dtype=torch.float16, device=qkv.device)
        check(self.lib.cb_attention_masked_f16(self.h, qkv.data_ptr(), out.data_ptr(), n, t, heads, d // heads, lengths.data_ptr(), _stream_ptr()),
              "cb_attention_masked_f16", self.h)  # fmt: skip
        return out

    def layernorm_post_(self, h: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
        """cb_layernorm_post_f16: h (fp32 [rows][d]) normalised in place; returns the fp16 copy."""
        rows, d = h.shape
        y = torch.empty((rows, d), dtype=torch.float16, device=h.device)
        check(self.lib.cb_layernorm_post_f16(self.h, h.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), rows, d, eps, _stream_ptr()),
              "cb_layernorm_post_f16", self.h)  # fmt: skip
        return y

    def text_embed(self, ids: torch.Tensor, word: torch.Tensor, pos: torch.Tensor, type_row: torch.Tensor) -> torch.Tensor:
        """cb_text_embed: int32 cuda ids [n][L] -> fp32 (word[id] + type) + pos[t], [n][L][d]."""
        n, L = ids.shape
        d = word.shape[1]
        h = torch.empty((n, L, d), dtype=torch.float32, device=ids.device)
        check(self.lib.cb_text_embed(self.h, ids.data_ptr(), word.data_ptr(), pos.data_ptr(), type_row.data_ptr(), h.data_ptr(), n, L, d,
                                     _stream_ptr()), "cb_text_embed", self.h)  # fmt: skip
        return h


_CONTEXTS: dict[int, Context] = {}


def get_context(device: int | None = None) -> Context:
    """Process-wide context per device (stages and models of one actor process share it)."""
    dev = torch.cuda.current_device() if (device is None and torch.cuda.is_available()) else int(device or 0)
    c = _CONTEXTS.get(dev)
    if c is None or c.h is None:
        c = _CONTEXTS[dev] = Context(dev)
    return c


def affine_score(ctx: Context, emb: torch.Tensor, w: torch.Tensor, b: float) -> torch.Tensor:
    n, d = emb.shape
    out = torch.empty((n,), dtype=torch.float32, device=emb.device)
    check(ctx.lib.cb_affine_score(ctx.h, emb.data_ptr(), w.data_ptr(), float(b), out.data_ptr(), n, d, _stream_ptr()), "cb_affine_score", ctx.h)
    return out


def _set_tensors(ctx: Context, set_tensor, h, weights: dict) -> None:
    """Upload every named array of `weights` as contiguous fp32 through `set_tensor`, one of the library's cb_*_set_tensor functions."""
    for name, arr in weights.items():
        a = np.ascontiguousarray(arr, dtype=np.float32)
        check(set_tensor(h, name.encode(), a.ctypes.data_as(C.POINTER(C.c_float)), a.size), f"{set_tensor.__name__}({name})", ctx.h)


class Pool:
    def __init__(self, buf: torch.Tensor, desc: SurfacePool):
        self.buf, self.desc = buf, desc  # keep the tensor alive while the descriptor is in use


class VitTower(_Handle):
    """cb_vit_* wrapper: weights in (fp32 numpy, names of include/curate_b200.h cb_vit_set_tensor), embeddings / scores out."""

    def __init__(self, ctx: Context, cfg: dict, weights: dict, max_batch: int = 256, aesthetic: tuple | None = None):
        self.ctx, self.lib = ctx, ctx.lib
        self.cfg = dict(cfg)
        c = VitCfg(cfg["image_size"], cfg["patch"], cfg["hidden"], cfg["layers"], cfg["heads"], cfg["mlp"], cfg["proj_dim"],
                   _lib.ACT_QUICK_GELU if cfg["act"] == "quick_gelu" else _lib.ACT_GELU_TANH,
                   _lib.ARCH_CLIP if cfg["arch"] == "clip" else _lib.ARCH_SIGLIP, cfg["ln_eps"])  # fmt: skip
        h = C.c_void_p()
        check(self.lib.cb_vit_create(ctx.h, C.byref(c), C.byref(h)), "cb_vit_create", ctx.h)
        self.h = h
        ctx._children.add(self)
        _set_tensors(ctx, self.lib.cb_vit_set_tensor, self.h, weights)
        self.out_dim = cfg["proj_dim"] or cfg["hidden"]
        self.has_aesthetic = False
        if aesthetic is not None:
            w, b = aesthetic
            w = np.ascontiguousarray(w, dtype=np.float32)
            check(self.lib.cb_vit_set_aesthetic(self.h, w.ctypes.data_as(C.POINTER(C.c_float)), w.size, float(b)), "cb_vit_set_aesthetic", ctx.h)
            self.has_aesthetic = True
        check(self.lib.cb_vit_finalize(self.h, max_batch), "cb_vit_finalize", ctx.h)
        self.k_pad = int(self.lib.cb_vit_k_pad(self.h))
        self.max_batch = max_batch

    def _destroy(self):
        self.lib.cb_vit_destroy(self.h)

    def forward_patches(self, patches: torch.Tensor, want_features: bool = False):
        n = patches.shape[0]
        dev = patches.device
        emb = torch.empty((n, self.out_dim), dtype=torch.float32, device=dev)
        feat = torch.empty((n, self.out_dim), dtype=torch.float32, device=dev) if want_features else None
        score = torch.empty((n,), dtype=torch.float32, device=dev) if self.has_aesthetic else None
        check(self.lib.cb_vit_forward(self.h, patches.data_ptr(), n, emb.data_ptr(), feat.data_ptr() if feat is not None else None,
                                      score.data_ptr() if score is not None else None, _stream_ptr()), "cb_vit_forward", self.ctx.h)  # fmt: skip
        return emb, feat, score

    def embed_pool(self, pool: Pool, slots=None, mean=CLIP_MEAN, std=CLIP_STD, want_features: bool = False):
        arr, ptr = self.ctx._slots(pool, slots)
        n, dev = len(arr), pool.buf.device
        emb = torch.empty((n, self.out_dim), dtype=torch.float32, device=dev)
        feat = torch.empty((n, self.out_dim), dtype=torch.float32, device=dev) if want_features else None
        score = torch.empty((n,), dtype=torch.float32, device=dev) if self.has_aesthetic else None
        check(self.lib.cb_vit_embed_surfaces(self.h, C.byref(pool.desc), ptr, n, _f3(mean), _f3(std), emb.data_ptr(),
                                             feat.data_ptr() if feat is not None else None, score.data_ptr() if score is not None else None,
                                             _stream_ptr()), "cb_vit_embed_surfaces", self.ctx.h)  # fmt: skip
        return emb, feat, score


class Iv2Tower(_Handle):
    """cb_iv2_* wrapper: weights in (fp32 numpy, names of include/curate_b200.h cb_iv2_set_tensor), clip embeddings out."""

    FIELDS = ("image_size", "patch", "frames", "hidden", "layers", "heads", "mlp", "clip_dim", "embed_dim", "rms_eps", "ln_eps")

    def __init__(self, ctx: Context, cfg: dict, weights: dict, max_clips: int = 8):
        self.ctx, self.lib = ctx, ctx.lib
        self.cfg = {k: cfg[k] for k in self.FIELDS}
        h = C.c_void_p()
        check(self.lib.cb_iv2_create(ctx.h, C.byref(Iv2Cfg(*[self.cfg[k] for k in self.FIELDS])), C.byref(h)), "cb_iv2_create", ctx.h)
        self.h = h
        ctx._children.add(self)
        _set_tensors(ctx, self.lib.cb_iv2_set_tensor, self.h, weights)
        check(self.lib.cb_iv2_finalize(self.h, max_clips), "cb_iv2_finalize", ctx.h)
        self.frames, self.embed_dim, self.max_clips = self.cfg["frames"], self.cfg["embed_dim"], max_clips

    def _destroy(self):
        self.lib.cb_iv2_destroy(self.h)

    def forward(self, tubes: torch.Tensor) -> torch.Tensor:
        """float32 cuda [n, frames, 3, S, S] -> unit-norm float32 cuda [n, embed_dim]."""
        s = self.cfg["image_size"]
        assert tubes.is_cuda and tubes.dtype == torch.float32 and tuple(tubes.shape[1:]) == (self.frames, 3, s, s), (tubes.dtype, tubes.shape)
        tubes = tubes.contiguous()
        out = torch.empty((tubes.shape[0], self.embed_dim), dtype=torch.float32, device=tubes.device)
        check(self.lib.cb_iv2_forward(self.h, tubes.data_ptr(), tubes.shape[0], out.data_ptr(), _stream_ptr()), "cb_iv2_forward", self.ctx.h)
        return out

    def embed_pool(self, pool: Pool, slots, mean=IMAGENET_MEAN, std=IMAGENET_STD) -> torch.Tensor:
        """Decoded frames -> unit-norm float32 cuda [n_clips, embed_dim]: `slots` holds n_clips * frames surface indices of `pool`,
        clip-major (repeats allowed).  Bitwise forward(video_tube(pool, S, S, slots).view(n_clips, frames, 3, S, S))."""
        arr, ptr = self.ctx._slots(pool, slots)
        if len(arr) % self.frames:
            raise ValueError(f"{len(arr)} slots are not whole clips of {self.frames} frames")
        n = len(arr) // self.frames
        out = torch.empty((n, self.embed_dim), dtype=torch.float32, device=pool.buf.device)
        check(self.lib.cb_iv2_embed_surfaces(self.h, C.byref(pool.desc), ptr, n, _f3(mean), _f3(std), out.data_ptr(), _stream_ptr()),
              "cb_iv2_embed_surfaces", self.ctx.h)  # fmt: skip
        return out


class Iv2TextTower(_Handle):
    """cb_iv2_text_* wrapper: weights in (fp32 numpy, names of include/curate_b200.h cb_iv2_text_set_tensor), text embeddings out."""

    FIELDS = ("hidden", "layers", "heads", "mlp", "vocab", "max_pos", "embed_dim", "ln_eps")

    def __init__(self, ctx: Context, cfg: dict, weights: dict, max_texts: int = 64, max_len: int = 40):
        self.ctx, self.lib = ctx, ctx.lib
        self.cfg = {k: cfg[k] for k in self.FIELDS}
        h = C.c_void_p()
        check(self.lib.cb_iv2_text_create(ctx.h, C.byref(Iv2TextCfg(*[self.cfg[k] for k in self.FIELDS])), C.byref(h)), "cb_iv2_text_create", ctx.h)
        self.h = h
        ctx._children.add(self)
        _set_tensors(ctx, self.lib.cb_iv2_text_set_tensor, self.h, weights)
        check(self.lib.cb_iv2_text_finalize(self.h, max_texts, max_len), "cb_iv2_text_finalize", ctx.h)
        self.embed_dim, self.max_texts, self.max_len = self.cfg["embed_dim"], max_texts, max_len

    def _destroy(self):
        self.lib.cb_iv2_text_destroy(self.h)

    def forward(self, ids: np.ndarray, lengths: np.ndarray) -> torch.Tensor:
        """Host int32 ids [n, L] and lengths [n] -> unit-norm float32 cuda [n, embed_dim]."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        lengths = np.ascontiguousarray(lengths, dtype=np.int32)
        assert ids.ndim == 2 and lengths.shape == (ids.shape[0],), (ids.shape, lengths.shape)
        n, L = ids.shape
        out = torch.empty((n, self.embed_dim), dtype=torch.float32, device=f"cuda:{self.ctx.device}")
        check(self.lib.cb_iv2_text_forward(self.h, ids.ctypes.data_as(C.POINTER(C.c_int32)), lengths.ctypes.data_as(C.POINTER(C.c_int32)), n, L,
                                           out.data_ptr(), _stream_ptr()), "cb_iv2_text_forward", self.ctx.h)  # fmt: skip
        return out


class ShotNet(_Handle):
    """cb_transnet_* wrapper: the reference state_dict in (its own key names), per-frame transition probabilities out."""

    UNUSED_KEYS = ("cls_layer2.weight", "cls_layer2.bias")  # many-hot head: built by the reference, never used by forward()

    def __init__(self, ctx: Context, state_dict: dict, max_windows: int = 16):
        self.ctx, self.lib = ctx, ctx.lib
        h = C.c_void_p()
        check(self.lib.cb_transnet_create(ctx.h, C.byref(h)), "cb_transnet_create", ctx.h)
        self.h = h
        ctx._children.add(self)
        weights = {name: arr.detach().cpu().numpy() if isinstance(arr, torch.Tensor) else arr for name, arr in state_dict.items()
                   if name not in self.UNUSED_KEYS and not name.endswith("num_batches_tracked")}  # fmt: skip
        _set_tensors(ctx, self.lib.cb_transnet_set_tensor, self.h, weights)
        check(self.lib.cb_transnet_finalize(self.h, max_windows), "cb_transnet_finalize", ctx.h)
        self.max_windows = max_windows

    def _destroy(self):
        self.lib.cb_transnet_destroy(self.h)

    def forward(self, windows: torch.Tensor) -> torch.Tensor:
        """uint8 cuda [B, T, 27, 48, 3] -> fp32 cuda [B, T, 1] (the reference model's call signature, transnetv2.py:569-580)."""
        assert windows.is_cuda and windows.dtype == torch.uint8 and windows.dim() == 5 and tuple(windows.shape[2:]) == (27, 48, 3), windows.shape
        windows = windows.contiguous()
        b, t = windows.shape[:2]
        out = torch.empty((b, t, 1), dtype=torch.float32, device=windows.device)
        check(self.lib.cb_transnet_forward(self.h, windows.data_ptr(), b, t, out.data_ptr(), _stream_ptr()), "cb_transnet_forward", self.ctx.h)
        return out

    def predict(self, frames: torch.Tensor) -> torch.Tensor:
        """uint8 cuda [n, 27, 48, 3] (a whole video) -> fp32 cuda [n] stitched probabilities."""
        assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and tuple(frames.shape[1:]) == (27, 48, 3), frames.shape
        frames = frames.contiguous()
        out = torch.empty((frames.shape[0],), dtype=torch.float32, device=frames.device)
        check(self.lib.cb_transnet_predict(self.h, frames.data_ptr(), frames.shape[0], out.data_ptr(), _stream_ptr()), "cb_transnet_predict", self.ctx.h)
        return out


# ---- demux + NVDEC ------------------------------------------------------------------------------------
def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
    return np.frombuffer(bytes(data) if not isinstance(data, (bytes, bytearray, memoryview)) else data, dtype=np.uint8)


def mp4_index(data, ctx: Context | None = None) -> dict:
    """cb_mp4_index: video-track facts + per-sample PTS ticks (decode order) + sync flags (host-only parse)."""
    buf = _as_u8(data)
    lib = ctx.lib if ctx is not None else _lib.load()
    h = ctx.h if ctx is not None else None
    info = _lib.Mp4Info()
    check(lib.cb_mp4_index(h, buf.ctypes.data, buf.size, C.byref(info), None, None, 0), "cb_mp4_index", h)
    n = info.n_samples
    pts = np.empty(n, dtype=np.int64)
    sync = np.empty(n, dtype=np.uint8)
    check(lib.cb_mp4_index(h, buf.ctypes.data, buf.size, C.byref(info), pts.ctypes.data_as(C.POINTER(C.c_int64)),
                           sync.ctypes.data_as(C.POINTER(C.c_uint8)), n), "cb_mp4_index", h)  # fmt: skip
    return {"codec": info.codec, "width": info.width, "height": info.height, "timescale": info.timescale, "n_samples": n,
            "n_sync": info.n_sync, "has_ctts": bool(info.has_ctts), "duration": info.duration, "sample_bytes": info.sample_bytes,
            "pts": pts, "sync": sync}  # fmt: skip


_NVDEC_OK: dict[int, bool] = {}


def nvdec_available(ctx: Context) -> bool:
    """cb_nvdec_probe, once per device: False where libnvcuvid loads but the driver reports no H.264 decode for this process
    (containers granted only the compute capability).  Decode requests then take the host path (host_decode.py: same pictures,
    same surface pools) after one warning; CURATE_B200_DECODE=nvdec makes that an error instead.  A missing libnvcuvid raises."""
    if ctx.device not in _NVDEC_OK:
        rc = ctx.lib.cb_nvdec_probe(ctx.h)
        if rc < 0:
            check(rc, "cb_nvdec_probe", ctx.h)
        if rc == 0:
            if os.environ.get("CURATE_B200_DECODE") == "nvdec":
                raise _lib.CurateB200Error(-4, "cb_nvdec_probe", "the driver reports no H.264 decode for this device and CURATE_B200_DECODE=nvdec")
            logger.warning(f"NVDEC of cuda:{ctx.device} is not usable from this process (cuvidGetDecoderCaps: no H.264 support): "
                           "clips are decoded on the HOST with libavcodec - far below the hardware decode rate")  # fmt: skip
        _NVDEC_OK[ctx.device] = rc == 1
    return _NVDEC_OK[ctx.device]


class Decoder(_Handle):
    """One decode session: NVDEC (cb_decoder_*), or libavcodec on the host where the device's NVDEC is not usable (nvdec_available).
    Not thread-safe: use one per host thread."""

    def __init__(self, ctx: Context):
        self.ctx, self.lib = ctx, ctx.lib
        self.host = not nvdec_available(ctx)
        if self.host:
            self.h = True
            return
        h = C.c_void_p()
        check(self.lib.cb_decoder_create(ctx.h, C.byref(h)), "cb_decoder_create", ctx.h)
        self.h = h
        ctx._children.add(self)

    def _destroy(self):
        if not self.host:
            self.lib.cb_decoder_destroy(self.h)

    def _host_decode(self, buf, ids, pool, slots, seek_keyframes: bool) -> dict:
        """decode() on the host: the same request checks and statistics as cb_decoder_decode_ex, pictures uploaded as NV12."""
        from . import host_decode

        idx = mp4_index(buf, self.ctx)  # CB_ERR_DEMUX on anything that is not an mp4 with a video track
        n = idx["n_samples"]
        w2, h2 = even_size(idx["width"], idx["height"])
        st = {"frames_decoded": 0, "frames_emitted": 0, "coded": ((idx["width"] + 15) & ~15, (idx["height"] + 15) & ~15), "size": (idx["width"], idx["height"])}
        if pool is not None and len(ids) == 0:
            return st
        if pool is not None:
            if np.any(np.diff(ids) < 0) or ids[0] < 0:
                raise _lib.CurateB200Error(-2, "cb_decoder_decode", "frame ids must be ascending")
            if ids[-1] >= n:
                raise _lib.CurateB200Error(-2, "cb_decoder_decode", f"frame id {ids[-1]} beyond the clip ({n} frames)")
            if (pool.desc.width, pool.desc.height) != (w2, h2):
                raise _lib.CurateB200Error(-4, "cb_decoder_decode", f"decode: pool is {pool.desc.width}x{pool.desc.height}, the stream {w2}x{h2}")
            if slots.min() < 0 or slots.max() >= pool.buf.shape[0]:
                raise _lib.CurateB200Error(-2, "cb_decoder_decode", "destination slot out of range")
        last = int(ids[-1]) if pool is not None else n - 1
        runs = [(0, last)]
        if seek_keyframes and pool is not None and not idx["has_ctts"]:  # no reordering: display index = sample index
            starts = np.flatnonzero(idx["sync"])
            gop = np.searchsorted(starts, ids, side="right") - 1
            runs = [(int(starts[g]), int(ids[gop == g].max())) for g in np.unique(gop)]
        where: dict[int, list[int]] = {}
        if pool is not None:
            for i, s in zip(ids.tolist(), slots.tolist()):
                where.setdefault(i, []).append(s)
        emitted = 0

        def on_frame(i, y, u, v):
            nonlocal emitted
            if i in where:
                _upload_yuv420(pool, where[i], y, u, v)
                emitted += len(where[i])

        try:
            st["frames_decoded"], _, _ = host_decode.decode(buf, idx["sync"], runs, on_frame)
        except ValueError as exc:
            raise _lib.CurateB200Error(-4, "cb_decoder_decode", f"decode: {exc}") from exc
        if pool is not None and emitted != len(ids):
            raise _lib.CurateB200Error(-4, "cb_decoder_decode", f"decode: {emitted} of {len(ids)} frames delivered")
        st["frames_emitted"] = emitted
        return st

    def decode(self, data, frame_ids, pool: Pool, dst_slots, seek_keyframes: bool = False) -> dict:
        """Decode `data` (mp4 bytes) and copy display-order frames `frame_ids` (ascending, repeats allowed)
        into `pool` slots `dst_slots`.  `seek_keyframes` skips GOPs that hold no wanted frame (identical output).
        Raises CurateB200Error on demux / decode failure."""
        buf = _as_u8(data)
        ids = np.ascontiguousarray(frame_ids, dtype=np.int32)
        slots = np.ascontiguousarray(dst_slots, dtype=np.int32)
        assert len(ids) == len(slots)
        if self.host:
            return self._host_decode(buf, ids, pool, slots, seek_keyframes)
        st = _lib.DecodeStats()
        flags = _lib.DECODE_SEEK_SYNC if seek_keyframes else 0
        check(self.lib.cb_decoder_decode_ex(self.h, buf.ctypes.data, buf.size, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids),
                                            C.byref(pool.desc), slots.ctypes.data_as(C.POINTER(C.c_int32)), flags, C.byref(st)),
              "cb_decoder_decode", self.ctx.h)  # fmt: skip
        return {"frames_decoded": st.frames_decoded, "frames_emitted": st.frames_emitted, "coded": (st.coded_width, st.coded_height),
                "size": (st.width, st.height)}  # fmt: skip


def _upload_yuv420(pool: Pool, slots, y: np.ndarray, u: np.ndarray, v: np.ndarray) -> None:
    """One decoded 4:2:0 picture as NV12 into `slots` of the pool (the layout NVDEC's mapped surfaces are copied into)."""
    rows, pitch = pool.buf.shape[1:]
    luma_rows = pool.desc.luma_rows
    nv12 = np.zeros((rows, pitch), dtype=np.uint8)
    nv12[: y.shape[0], : y.shape[1]] = y
    nv12[luma_rows : luma_rows + u.shape[0], 0 : 2 * u.shape[1] : 2] = u
    nv12[luma_rows : luma_rows + v.shape[0], 1 : 2 * v.shape[1] : 2] = v
    t = torch.from_numpy(nv12).to(pool.buf.device)
    for s in slots:
        pool.buf[s].copy_(t)


def decode_discard(dec: Decoder, data) -> int:
    """Decode every picture of the clip and deliver none; returns the number decoded (NVDEC ceiling measurement)."""
    buf = _as_u8(data)
    if dec.host:
        return dec._host_decode(buf, None, None, None, False)["frames_decoded"]
    st = _lib.DecodeStats()
    check(dec.lib.cb_decoder_decode_ex(dec.h, buf.ctypes.data, buf.size, None, 0, None, None, _lib.DECODE_DISCARD_ALL, C.byref(st)),
          "cb_decoder_decode_ex", dec.ctx.h)
    return st.frames_decoded


def decode_thumbnails(dec: Decoder, data, out_w: int, out_h: int, n_frames: int) -> torch.Tensor:
    """Every frame of the clip as uint8 cuda [n, out_h, out_w, 3] (cb_decoder_decode_thumbnails)."""
    buf = _as_u8(data)
    if dec.host:  # one decode pass; a batch of frames at a time through a surface pool and the same bilinear kernel
        from . import host_decode

        idx = mp4_index(buf, dec.ctx)
        n, batch, parts = min(n_frames, idx["n_samples"]), 64, []
        pool = alloc_nv12_pool(dec.ctx, batch, idx["width"], idx["height"])

        def on_frame(i, y, u, v):
            _upload_yuv420(pool, [i % batch], y, u, v)
            if i % batch == batch - 1 or i == n - 1:
                parts.append(dec.ctx.preprocess_bilinear_u8(pool, out_w, out_h, slots=np.arange(i % batch + 1, dtype=np.int32)))

        try:
            host_decode.decode(buf, idx["sync"], [(0, n - 1)], on_frame)
        except ValueError as exc:
            raise _lib.CurateB200Error(-4, "cb_decoder_decode_thumbnails", f"decode: {exc}") from exc
        return torch.cat(parts) if parts else torch.empty((0, out_h, out_w, 3), dtype=torch.uint8, device=f"cuda:{dec.ctx.device}")
    out = torch.empty((n_frames, out_h, out_w, 3), dtype=torch.uint8, device=f"cuda:{dec.ctx.device}")
    st = _lib.DecodeStats()
    check(dec.lib.cb_decoder_decode_thumbnails(dec.h, buf.ctypes.data, buf.size, out_w, out_h, out.data_ptr(), n_frames, C.byref(st)),
          "cb_decoder_decode_thumbnails", dec.ctx.h)  # fmt: skip
    return out[: st.frames_emitted]


def alloc_nv12_pool(ctx: Context, slots: int, width: int, height: int, colour: str = "opencv") -> Pool:
    """Device NV12 surface pool for `slots` frames of width x height (pitch aligned to 256 bytes); `colour` as Context.nv12_pool."""
    w2, h2 = even_size(width, height)
    pitch = (w2 + 255) // 256 * 256
    buf = torch.empty((slots, h2 + h2 // 2, pitch), dtype=torch.uint8, device=f"cuda:{ctx.device}")
    return ctx.nv12_pool(buf, w2, h2, h2, colour)


# ---- host placement + persistent NVDEC sessions ---------------------------------------------------------
def _parse_cpulist(text: str) -> set[int]:
    out: set[int] = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        out.update(range(int(lo), int(hi or lo) + 1))
    return out


def device_numa_cpus(ctx: Context) -> tuple[int | None, list[int]]:
    """(NUMA node of the context's GPU, host CPUs of that node this process may run on).  ([] when the topology is not
    visible - e.g. numa_node = -1 on single-socket hosts - in which case nothing is pinned.)"""
    import os

    buf = C.create_string_buffer(32)
    try:
        check(ctx.lib.cb_device_pci_bus_id(ctx.h, buf, 32), "cb_device_pci_bus_id", ctx.h)
        bus = buf.value.decode().lower()
        with open(f"/sys/bus/pci/devices/{bus}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None, []
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read())
        return node, sorted(cpus & os.sched_getaffinity(0))
    except (OSError, ValueError, _lib.CurateB200Error):
        return None, []


class ShapeCache:
    """One object per stream shape (any hashable, normally (width, height)), made by `create(shape)` on first use.  At most
    MAX_SHAPES are kept: a new shape beyond that hands the least recently used object to `close`."""

    MAX_SHAPES = 4

    def __init__(self, create, close):
        self._create, self._close = create, close
        self._items: dict = {}  # least recently used first

    def get(self, shape):
        v = self._items.pop(shape, None)
        if v is None:
            while len(self._items) >= self.MAX_SHAPES:
                self._close(self._items.pop(next(iter(self._items))))
            v = self._create(shape)
        self._items[shape] = v
        return v

    def values(self) -> list:
        return list(self._items.values())

    def close(self) -> None:
        for v in self._items.values():
            self._close(v)
        self._items.clear()


class SessionTable(ShapeCache):
    """One NVDEC session per stream shape for a single-threaded caller (DecoderPool keeps one table per worker thread): a
    session that is fed another resolution is destroyed and re-created by the driver, ~0.4 s each time."""

    def __init__(self, ctx: Context):
        super().__init__(lambda shape: Decoder(ctx), Decoder.close)
        self.ctx = ctx


class SurfacePools:
    """A stage's NV12 decode surfaces: per stream size (a ShapeCache) a ring of `depth` pools, so that decode into one pool
    overlaps the kernels that read another.  A pool holds the smallest min_slots * 2^k slots that fit the request; a pool
    that is too small is dropped before its replacement is allocated."""

    def __init__(self, ctx: Context, depth: int, min_slots: int, colour: str):
        self.ctx, self.min_slots, self.colour = ctx, min_slots, colour
        self._rings = ShapeCache(lambda size: [None] * depth, list.clear)

    def get(self, size: tuple[int, int], n: int, r: int = 0) -> Pool:
        """Pool `r` of the ring for streams of `size` = (width, height), with at least `n` slots."""
        ring = self._rings.get(size)
        cap = self.min_slots
        while cap < n:
            cap *= 2
        if ring[r] is None or ring[r].buf.shape[0] < cap:
            ring[r] = None
            ring[r] = alloc_nv12_pool(self.ctx, cap, size[0], size[1], self.colour)
        return ring[r]

    def clear(self) -> None:
        self._rings.close()


class DecoderPool:
    """Persistent NVDEC sessions behind a thread pool: one `SessionTable` per worker thread, created on first use and kept
    across calls (session creation costs ~10 ms and a context-lock round trip), worker threads pinned to the host CPUs of the
    GPU's NUMA node (bitstream parsing + H2D staging are host work: on a two-socket 8-GPU box the far socket costs decode rate)."""

    MAX_SHAPES = SessionTable.MAX_SHAPES  # sessions a worker thread keeps

    def __init__(self, ctx: Context, sessions: int, pin: bool = True):
        import threading
        from concurrent.futures import ThreadPoolExecutor

        self.ctx, self.sessions = ctx, int(sessions)
        self.numa_node, cpus = device_numa_cpus(ctx) if pin else (None, [])
        self.cpus = cpus
        self._tls = threading.local()
        self._tables: list[SessionTable] = []
        self._lock = threading.Lock()
        self._tp = ThreadPoolExecutor(max_workers=self.sessions, thread_name_prefix="cb-nvdec", initializer=self._init_thread)

    def _init_thread(self) -> None:
        import os

        if self.cpus:
            try:
                os.sched_setaffinity(0, self.cpus)  # pid 0 = the calling thread
            except OSError:
                pass

    def decoder(self, shape=None) -> Decoder:
        """This thread's session for streams of `shape` (any hashable, normally (width, height)).  A cuvid decoder is bound to
        one coded size: feeding a session a clip of another resolution destroys and re-creates it (hundreds of ms, serialised
        in the driver - measured: a 720p / 1080p / 4K mix ran 4-12x below the NVDEC rate with one session per thread), so a
        thread keeps one session per shape instead."""
        table = getattr(self._tls, "table", None)
        if table is None:
            table = self._tls.table = SessionTable(self.ctx)
            with self._lock:
                self._tables.append(table)
        return table.get(shape)

    @property
    def _decoders(self) -> list[Decoder]:
        """The open sessions of every worker thread."""
        with self._lock:
            return [d for t in self._tables for d in t.values()]

    def submit(self, fn, *args, shape=None, **kw):
        """fn(decoder, *args, **kw) on a pool thread with that thread's own session (for streams of `shape`, see decoder())."""
        return self._tp.submit(lambda: fn(self.decoder(shape), *args, **kw))

    def submit_group(self, pool: Pool, shape, jobs, seek_keyframes: bool = False) -> list:
        """Decode each (data, frame ids) job into `pool`, the jobs' frames in consecutive slots from slot 0, on sessions for
        streams of `shape`.  -> [(first slot of the job, future of its Decoder.decode statistics)] in job order."""
        def decode(dec, data, ids, slots):
            return dec.decode(data, ids, pool, slots, seek_keyframes=seek_keyframes)

        out, first = [], 0
        for data, ids in jobs:
            out.append((first, self.submit(decode, data, ids, np.arange(first, first + len(ids), dtype=np.int32), shape=shape)))
            first += len(ids)
        return out

    def close(self) -> None:
        self._tp.shutdown(wait=True)
        with self._lock:
            for t in self._tables:
                t.close()
            self._tables.clear()


def collect_group(jobs) -> tuple[int, list]:
    """Wait for the jobs of DecoderPool.submit_group -> (frames decoded by the jobs that succeeded, summed; per job its
    CurateB200Error or None, in job order)."""
    decoded, errs = 0, []
    for _, fut in jobs:
        try:
            decoded += fut.result()["frames_decoded"]
            errs.append(None)
        except _lib.CurateB200Error as e:
            errs.append(e)
    return decoded, errs


def run_decode_groups(items, plan, pools: SurfacePools, decoders, compute, *, on_error, max_frames: int, on_short=None, depth: int = 2,
                      seek_keyframes: bool = False) -> tuple[int, int]:  # fmt: skip
    """Decode the kept frames of clips [(clip, mp4 bytes)] into surface pools, group by group, and hand each group to `compute`.

    plan(clip, data) gives (surface size, ascending frame ids to decode, slot of every kept frame relative to the clip's first slot).
    It raises CurateB200Error / ValueError for a clip that goes to on_error(clip, e); a plan that can return None (too few frames)
    needs on_short(clip).  A clip keeping more than `max_frames` frames goes to on_error; the others are grouped per surface size, in the
    order sizes are first seen, each group filled with whole clips up to `max_frames` kept frames.  Group k is decoded by decoders()
    (a DecoderPool) into pool k % depth (depth >= 2) of its size's ring while the groups before it compute.

    compute(k, pool, ok, slots) gets the clips whose decode succeeded as [(clip, number of kept frames)] (the others go to on_error)
    and their kept frames' surface indices, concatenated clip-major.  It queues the GPU work that reads the pool and returns None or
    a finisher that writes the results onto the clips.  Per group k: wait for its decode, compute(k) and record an event, wait on
    group k - 1's event, submit group k + depth - 1, run group k - 1's finisher.  The GPU has group k queued while the host writes
    k - 1's results and submits decode, and since a size's groups are contiguous, the last reader of the pool that group
    k + depth - 1 decodes into is group k - 1 at the latest.  -> (frames decoded, groups)."""
    by_size: dict[tuple, list] = {}
    for clip, data in items:
        try:
            planned = plan(clip, data)
        except (_lib.CurateB200Error, ValueError) as e:
            on_error(clip, e)
            continue
        if planned is None:
            on_short(clip)
            continue
        size, ids, inverse = planned
        if len(inverse) > max_frames:
            on_error(clip, ValueError(f"{len(inverse)} kept frames exceed max_frames={max_frames}"))
            continue
        by_size.setdefault(size, []).append((clip, data, ids, inverse))
    groups: list[tuple[tuple, list]] = []
    for size, clips in by_size.items():
        used = max_frames
        for c in clips:
            if used + len(c[3]) > max_frames:
                groups.append((size, []))
                used = 0
            groups[-1][1].append(c)
            used += len(c[3])
    ring_pos: dict[tuple, int] = {}
    pending: dict[int, tuple] = {}

    def submit(k):
        size, clips = groups[k]
        r = ring_pos.get(size, 0)
        ring_pos[size] = (r + 1) % depth
        pool = pools.get(size, sum(len(ids) for _, _, ids, _ in clips), r)
        pending[k] = pool, decoders().submit_group(pool, size, [(data, ids) for _, data, ids, _ in clips], seek_keyframes)

    decoded, prev_event, prev_finisher = 0, None, None  # of group k - 1
    for k in range(min(depth - 1, len(groups))):
        submit(k)
    for k, (_, clips) in enumerate(groups):
        pool, jobs = pending.pop(k)
        n, errs = collect_group(jobs)
        decoded += n
        ok, slots = [], []
        for (clip, _, _, inverse), (first, _), err in zip(clips, jobs, errs):
            if err is not None:
                on_error(clip, err)
                continue
            ok.append((clip, len(inverse)))
            slots.append(first + inverse)
        finisher = compute(k, pool, ok, np.concatenate(slots).astype(np.int32)) if ok else None
        event = torch.cuda.Event()
        event.record(torch.cuda.current_stream())
        if prev_event is not None:
            prev_event.synchronize()
        if k + depth - 1 < len(groups):
            submit(k + depth - 1)
        if prev_finisher is not None:
            prev_finisher()
        prev_event, prev_finisher = event, finisher
    if prev_event is not None:
        prev_event.synchronize()
        if prev_finisher is not None:
            prev_finisher()
    return decoded, len(groups)
