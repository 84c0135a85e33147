"""Oracle: the host plans of the two CLIP resample kernels (csrc/preprocess.cu, csrc/preprocess_tc.cu), restated in Python.

`run_clip_preprocess` turns (width, height, surface format, res) into a plan before it launches anything:

* torchvision's size and crop rules give the resized size and the crop offsets, and `oracle.preprocess.aa_bicubic_taps` the tap tables
  of the cropped outputs;
* more than 64 taps on an axis (or an odd NV12 size) is CB_ERR_UNSUPPORTED;
* the tensor-pipe kernel (`clip_preprocess_tc_kernel`) takes NV12 pools with at most 40 vertical taps whose geometry fits: 32-column
  slabs, or 16 when a 32-column slab's source window exceeds one 256-byte TMA box; `ru` source rows per unit from the tap count;
  at most kMaxUnits units; shared memory;
* everything else runs the SIMT kernel (`clip_preprocess_simt_kernel`): column tile 32 -> 16 -> 8 until the strip window fits one
  TMA box, a union window per group of 4 columns, a ring of filtered rows and its shared-memory carve-up.

`plan()` returns the fields of `cb_preprocess_plan_info`, so the GPU tests compare the library's own plan with this one field by field.
The kernels' constants are read back out of the sources (`constants_from_source`).  `plan_class()` names the class of a point, `sweep()`
lists the points the tests run, chosen so that every class and both sides of every boundary are reached, and `constant_*` build inputs
whose exact answer is known.

Test infrastructure only (see oracle/__init__.py).
"""

from __future__ import annotations

import functools
import re
from pathlib import Path

import numpy as np

from . import color
from .preprocess import aa_bicubic_taps, center_crop_offsets, resized_output_size

CSRC = Path(__file__).resolve().parent.parent / "cosmos_curate_b200" / "csrc"
FORMATS = ("opencv", "swscale", "rgb")  # CB_FMT_NV12, CB_FMT_NV12_SWS, CB_FMT_RGB24
FMT_CODE = {"opencv": 0, "rgb": 1, "swscale": 2}
PRE_NONE, PRE_TC, PRE_SIMT = 0, 1, 2
WHY = ("OK", "RGB", "TAPS40", "KW", "RU", "UNITS", "SMEM", "TAPS64", "SWA", "ODD")  # CB_PRE_WHY_* by value
W = {name: i for i, name in enumerate(WHY)}

# The values the sources hold (checked against them by constants_from_source in tests/test_preprocess_plan_cpu.py).
K = {
    "kNC": 32, "kRingRows": 64, "kRingStride": 100, "kMaxUnits": 128, "kVRows": 16, "kVTaps": 40, "kSR": 32,
    "tc_max_taps": 40, "max_taps": 64, "ru_max": 40, "box_bytes": 256, "x_align": 16, "simt_ring_min": 64, "smem_max": 227 * 1024,
}  # fmt: skip


def _one(pattern: str, text: str, where: str) -> str:
    m = re.findall(pattern, text)
    assert len(m) >= 1, f"{where}: no match for {pattern!r}"
    assert len(set(m)) == 1, f"{where}: {pattern!r} matches different values {m}"
    return m[0]


def constants_from_source() -> dict:
    """K as preprocess_tc.cu and preprocess.cu write it: the constexprs, the 40- and 64-tap limits, the 256-byte box in every window test,
    the SIMT x alignment and ring start, the 227 KB shared-memory limit."""
    tc, simt = (CSRC / "preprocess_tc.cu").read_text(), (CSRC / "preprocess.cu").read_text()
    env: dict[str, int] = {}
    for decl in re.findall(r"constexpr int (k\w+ = [^;]+);", tc):
        for item in re.split(r",\s*(?=k\w+ = )", decl):  # `constexpr int kVRows = 16, kVTaps = 40;`
            name, expr = item.split(" = ", 1)
            env[name] = int(eval(expr, {"__builtins__": {}}, dict(env)))  # noqa: S307 - integer constexprs of our own source
    out = {k: env[k] for k in ("kNC", "kRingRows", "kRingStride", "kMaxUnits", "kVRows", "kVTaps")}
    out["kSR"] = int(_one(r"constexpr int kSR = (\d+);", simt, "preprocess.cu"))
    out["tc_max_taps"] = int(_one(r"if \(ty->max_taps > (\d+)\) return 1;", tc, "preprocess_tc.cu"))
    lim = re.findall(r"if \(ty->max_taps > (\d+) \|\| tx->max_taps > (\d+)\)", simt)
    assert len(lim) == 1 and lim[0][0] == lim[0][1], lim
    out["max_taps"] = int(lim[0][0])
    plan_lim = re.findall(r"if \(tx\.max_taps > (\d+) \|\| ty\.max_taps > (\d+)\)", simt)
    assert plan_lim == lim, (plan_lim, lim)  # cb_preprocess_plan states the same limit
    out["ru_max"] = int(_one(r"p\.ru = std::min\((\d+), kRingRows - ty\.max_taps \+ 1\) & ~7;", tc, "preprocess_tc.cu"))
    boxes = re.findall(r"kw <= (\d+)\) break;", tc) + re.findall(r"p\.kw > (\d+)", tc) + re.findall(r"span <= (\d+) \|\|", simt) + re.findall(
        r"a\.swa > (\d+) \?", simt)  # fmt: skip
    assert len(boxes) == 4 and len(set(boxes)) == 1, boxes
    out["box_bytes"] = int(boxes[0])
    out["x_align"] = int(_one(r"a\.x_align = (\d+);", simt, "preprocess.cu"))
    out["simt_ring_min"] = int(_one(r"int ring = (\d+);", simt, "preprocess.cu"))
    smem = set(re.findall(r"smem > (\d+) \* 1024", tc + simt))
    assert len(smem) == 1, smem
    out["smem_max"] = int(smem.pop()) * 1024
    return out


# ------------------------------------------------------------------------------------------------ taps and plans
@functools.lru_cache(maxsize=4096)
def _axis_taps(in_size: int, out_size: int, crop_off: int, crop_len: int):
    xmin, xsize, w = aa_bicubic_taps(in_size, out_size)
    xmin, xsize = xmin[crop_off : crop_off + crop_len], xsize[crop_off : crop_off + crop_len]
    t = int(xsize.max())
    return xmin, xsize, np.ascontiguousarray(w[crop_off : crop_off + crop_len, :t]), t, int(xmin.min()), int((xmin + xsize).max())


def cropped_taps(width: int, height: int, res: int):
    """(new_w, new_h, top, left, taps_x, taps_y) where taps_* = (xmin, xsize, w, max_taps, src_begin, src_end) of the cropped outputs."""
    new_h, new_w = resized_output_size(height, width, res)
    top, left = center_crop_offsets(new_h, new_w, res)
    return new_w, new_h, top, left, _axis_taps(width, new_w, left, res), _axis_taps(height, new_h, top, res)


def tc_geometry(tx, ty, res: int) -> dict:
    """preprocess_tc.cu tc_geometry: slab width, windows, k-steps of the two N-tiles, rows per unit, units, shared memory, why."""
    xmin, xsize, _, _, _, _ = tx
    _, _, _, ty_taps, y_begin_src, y_end_src = ty
    hi_all = xmin + xsize
    for nc in (K["kNC"], 16):
        n_slabs = (res + nc - 1) // nc
        x_lo, k0, nk = [0] * n_slabs, [0] * (2 * n_slabs), [0] * (2 * n_slabs)
        kw = kbmax = 0
        for s in range(n_slabs):
            c0, c1 = s * nc, min(res, s * nc + nc)
            x_lo[s] = int(xmin[c0]) & ~15
            kw = max(kw, int(hi_all[c0:c1].max()) - x_lo[s])
            for j in range(2):
                t0, t1 = c0 + 16 * j, min(c1, c0 + 16 * j + 16)
                if t0 >= t1:
                    continue
                first = (int(xmin[t0]) - x_lo[s]) // 16
                end = int(hi_all[t0:t1].max()) - x_lo[s]
                k0[2 * s + j], nk[2 * s + j] = first, (end - first * 16 + 15) // 16
                kbmax = max(kbmax, nk[2 * s + j] * 16)
        if kw <= K["box_bytes"]:
            break
    kw_raw = kw
    kw, kb = (kw + 63) & ~63, (kbmax + 63) & ~63
    ru = min(K["ru_max"], K["kRingRows"] - ty_taps + 1) & ~7
    y_begin = y_begin_src & ~1
    n_units = (y_end_src - y_begin + ru - 1) // ru if ru > 0 else 0
    b_tile = (kb // 64) * 4096
    smem = (1024 + kw * 256 + 2 * b_tile + (((ru + ru // 2) * kw + 127) & ~127)
            + (K["kRingRows"] * K["kRingStride"] + K["kVRows"] * K["kVTaps"] + 2 * K["kVRows"] + K["kMaxUnits"]) * 4 + 64)  # fmt: skip
    why = ("KW" if kw > K["box_bytes"] else "RU" if ru < 16 else "UNITS" if n_units > K["kMaxUnits"] else "SMEM" if smem > K["smem_max"]
           else "OK")  # fmt: skip
    return {"nc": nc, "n_slabs": n_slabs, "kw": kw, "kb": kb, "ru": ru, "n_units": n_units, "y_begin": y_begin, "smem": smem, "why": why,
            "kw_raw": kw_raw, "x_lo": x_lo, "k0": k0, "nk": nk}  # fmt: skip


def simt_geometry(tx, ty, res: int, fmt: str) -> dict:
    """preprocess.cu simt_geometry: column tile, strip window, union window, ring, strips, shared memory, why."""
    xmin, xsize, _, _, _, _ = tx
    _, _, _, ty_taps, y_begin_src, y_end_src = ty
    kSR, align = K["kSR"], K["x_align"]
    y_begin = y_begin_src & ~1
    n_strips = (y_end_src - y_begin + kSR - 1) // kSR
    ring = K["simt_ring_min"]
    while ring < kSR + ty_taps:
        ring <<= 1
    hi_all = xmin + xsize
    spans = {}
    tc = 32
    while True:
        tiles = (res + tc - 1) // tc
        span = max(int(hi_all[t * tc : min(res, t * tc + tc)].max()) - (int(xmin[t * tc]) & ~(align - 1)) for t in range(tiles))
        spans[tc] = span
        if span <= K["box_bytes"] or tc == 8:
            break
        tc //= 2
    swa = (span + 15) & ~15
    gu = 1
    for c in range(0, res, 4):
        if (c % tc) + 4 > tc and (c % tc) % 4:
            continue
        cl = min(res, c + 4, (c // tc + 1) * tc)
        gu = max(gu, int((hi_all[c:cl] - xmin[c]).max()))
    raw_stage = swa * kSR * 3 // 2 if fmt != "rgb" else 3 * swa * kSR
    groups = (tc + 3) // 4
    smem = 2 * raw_stage + 3 * kSR * (swa + 1) * 4 + 3 * ring * (tc | 1) * 4 + groups * gu * 16 + 2 * groups * 4 + 80
    why = "SWA" if swa > K["box_bytes"] else "SMEM" if smem > K["smem_max"] else "OK"
    return {"tc": tc, "tiles": tiles, "swa": swa, "gu": gu, "ring": ring, "n_strips": n_strips, "y_begin": y_begin, "smem": smem, "why": why,
            "spans": spans}  # fmt: skip


FIELDS = ("kernel", "simt_kernel", "tc_why", "simt_why", "new_w", "new_h", "top", "left", "taps_x", "taps_y", "src_y_begin", "src_y_end",
          "tc_nc", "tc_n_slabs", "tc_kw", "tc_kb", "tc_ru", "tc_n_units", "tc_y_begin", "tc_smem",
          "simt_tc", "simt_tiles", "simt_swa", "simt_gu", "simt_ring", "simt_n_strips", "simt_y_begin", "simt_smem")  # fmt: skip


@functools.lru_cache(maxsize=4096)
def _plan(width: int, height: int, fmt: str, res: int):
    nv12 = fmt != "rgb"
    new_h, new_w = resized_output_size(height, width, res)
    top, left = center_crop_offsets(new_h, new_w, res)
    out = dict.fromkeys(FIELDS, 0)
    out.update(new_w=new_w, new_h=new_h, top=top, left=left)
    if nv12 and (width | height) & 1:
        out.update(kernel=PRE_NONE, simt_kernel=PRE_NONE, tc_why=W["ODD"], simt_why=W["ODD"])
        return out, None, None
    _, _, _, _, tx, ty = cropped_taps(width, height, res)
    out.update(taps_x=tx[3], taps_y=ty[3], src_y_begin=ty[4], src_y_end=ty[5])
    if tx[3] > K["max_taps"] or ty[3] > K["max_taps"]:
        out.update(kernel=PRE_NONE, simt_kernel=PRE_NONE, tc_why=W["TAPS64"], simt_why=W["TAPS64"])
        return out, None, None
    t, s = tc_geometry(tx, ty, res), simt_geometry(tx, ty, res, fmt)
    out.update({f"tc_{k}": t[k] for k in ("nc", "n_slabs", "kw", "kb", "ru", "n_units", "y_begin", "smem")})
    out.update({f"simt_{k}": s[k] for k in ("tc", "tiles", "swa", "gu", "ring", "n_strips", "y_begin", "smem")})
    out["tc_why"] = W["RGB"] if not nv12 else W["TAPS40"] if ty[3] > K["tc_max_taps"] else W[t["why"]]
    out["simt_why"] = W[s["why"]]
    out["simt_kernel"] = PRE_SIMT if s["why"] == "OK" else PRE_NONE
    out["kernel"] = PRE_TC if out["tc_why"] == W["OK"] else out["simt_kernel"]
    return out, t, s


def plan(width: int, height: int, fmt: str, res: int) -> dict:
    """The fields of cb_preprocess_plan_info for a width x height pool of `fmt` ("opencv", "swscale" or "rgb") at `res`."""
    return dict(_plan(width, height, fmt, res)[0])


# ------------------------------------------------------------------------------------------------ classes
def _band(taps: int) -> str:
    return "<=25" if taps <= 25 else "26-33" if taps <= 33 else "34-40" if taps <= 40 else "41-64" if taps <= 64 else ">64"


def plan_class(width: int, height: int, fmt: str, res: int) -> dict:
    """The plan class of a point: which kernel runs (default and forced SIMT), why the other declines, the slab and tile widths, the
    vertical taps band (ru 40 / 32 / 24 of the tensor pipe, 41-64 SIMT only, > 64 refused), a partial last slab (with an empty second
    N-tile) or tile, up- or downscale per axis, the parity of the crop offsets and of the first source row, whether a source row is a
    whole number of 16-byte units, and the orientation."""
    p, t, s = _plan(width, height, fmt, res)
    bpp = 3 if fmt == "rgb" else 1
    c = {
        "kernel": ("none", "tc", "simt")[p["kernel"]], "simt_kernel": ("none", "tc", "simt")[p["simt_kernel"]],
        "tc_why": WHY[p["tc_why"]], "simt_why": WHY[p["simt_why"]], "fmt": fmt,
        "orientation": "landscape" if width > height else "portrait" if width < height else "square",
        "row_bytes_16": (width * bpp) % 16 == 0,
        "scale_x": "up" if p["new_w"] > width else "same" if p["new_w"] == width else "down",
        "scale_y": "up" if p["new_h"] > height else "same" if p["new_h"] == height else "down",
        "top_odd": p["top"] % 2 == 1, "left_odd": p["left"] % 2 == 1, "src_y_begin_odd": p["src_y_begin"] % 2 == 1,
        "res_mod32": res % 32,
    }  # fmt: skip
    if t is not None:
        c["taps_band"] = _band(p["taps_y"])
        c["tc_nc"], c["tc_ru"] = t["nc"], t["ru"]
        c["tc_partial_slab"] = res % t["nc"] != 0
        c["tc_empty_ntile"] = any(t["nk"][2 * k + 1] == 0 for k in range(t["n_slabs"])) if t["nc"] == 32 else False
        c["tc_partial_ntile"] = t["nc"] == 32 and res % 32 > 16  # the last slab's second N-tile has 1..15 columns
        c["simt_tc"] = s["tc"]
        c["simt_partial_tile"] = res % s["tc"] != 0
    else:
        c["taps_band"] = _band(max(p["taps_x"], p["taps_y"])) if p["taps_x"] else "odd"
    return c


# ------------------------------------------------------------------------------------------------ the sweep
SOURCES = ((96, 64), (160, 120), (222, 222), (224, 224), (226, 226), (426, 240), (448, 448), (640, 360), (854, 480), (1280, 720),
           (1440, 1080), (1920, 800), (1920, 1080), (1080, 1920), (2560, 1440), (2704, 1520), (2880, 1620), (3840, 1600), (3840, 2160),
           (2160, 3840), (4096, 2160), (5312, 2988), (6144, 3456))  # fmt: skip
RGB_ODD = ((853, 479), (641, 361), (1279, 719))  # RGB frames whose rows are not a whole number of 16-byte units
RESES = (224, 336, 384, 200)
# the sources also run at 336, 384 and 200: one of each size class, landscape and portrait
OTHER_RES_SOURCES = ((96, 64), (222, 222), (426, 240), (854, 480), (1280, 720), (1920, 1080), (1080, 1920), (2704, 1520), (3840, 2160),
                     (5312, 2988))  # fmt: skip
REFUSED = ((7680, 4320, 224),)  # 78 taps: CB_ERR_UNSUPPORTED


def _metric(width: int, height: int, res: int, name: str) -> int:
    p, t, s = _plan(width, height, "opencv", res)
    if name == "taps":
        return max(p["taps_x"], p["taps_y"])
    if t is None:
        return 10**9
    if name == "kw32":  # the widest 32-column slab window (before the 16-column fallback)
        _, _, _, _, tx, ty = cropped_taps(width, height, res)
        return tc_geometry_nc(tx, res, 32)
    if name == "span32":
        return s["spans"][32]
    if name == "span16":  # only where the 32-column tile was too wide
        return s["spans"].get(16, 10**9)
    raise KeyError(name)


def tc_geometry_nc(tx, res: int, nc: int) -> int:
    """The widest raw slab window at slab width nc."""
    xmin, xsize = tx[0], tx[1]
    hi = xmin + xsize
    return max(int(hi[c0 : min(res, c0 + nc)].max()) - (int(xmin[c0]) & ~15) for c0 in range(0, res, nc))


# class boundaries: (name, metric, threshold): a point with metric <= threshold and one with metric > threshold
BOUNDARIES = (("kw 256/257", "kw32", 256), ("swa 256/257 at 32 columns", "span32", 256),
              ("swa 256/257 at 16 columns", "span16", 256), ("taps 25/26", "taps", 25),
              ("taps 33/34", "taps", 33), ("taps 40/41", "taps", 40), ("taps 64/65", "taps", 64))  # fmt: skip


@functools.lru_cache(maxsize=None)
def boundary_points(res: int = 224) -> tuple:
    """For each boundary: (name, threshold, (metric, width, height) of the 16:9 NV12 source with the largest metric <= threshold,
    the same with the smallest metric > threshold).  Scans heights in steps of 2, width round(16 h / 9) made even."""
    cands = []
    for h in range(res + 2, 4600, 2):
        w = int(round(h * 16 / 9)) & ~1
        cands.append((w, h))
    out = []
    for name, metric, thr in BOUNDARIES:
        best_lo = best_hi = None
        for w, h in cands:
            m = _metric(w, h, res, metric)
            if m >= 10**9:
                continue
            if m <= thr and (best_lo is None or m > best_lo[0]):
                best_lo = (m, w, h)
            if m > thr and (best_hi is None or m < best_hi[0]):
                best_hi = (m, w, h)
        out.append((name, thr, best_lo, best_hi))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def sweep() -> tuple:
    """(width, height, formats, res) of every swept point.  NV12 sources run in both colour arithmetics and as RGB frames; the odd
    RGB sources as RGB only."""
    pts = []
    for w, h in SOURCES:
        pts.append((w, h, FORMATS, 224))
    for r in RESES[1:]:
        for w, h in OTHER_RES_SOURCES:
            pts.append((w, h, FORMATS, r))
    for w, h in RGB_ODD:
        pts.append((w, h, ("rgb",), 224))
        pts.append((w, h, ("rgb",), 200))
    # res 250: a partial last 32-column slab whose second N-tile is partial but not empty
    for w, h in ((854, 480), (1920, 1080), (1080, 1920), (2560, 1440)):
        pts.append((w, h, FORMATS, 250))
    # 5.3K at 201 (60 taps): the 8-column SIMT tile with a partial last tile
    pts.append((5312, 2988, FORMATS, 201))
    # a 6K portrait at 384 (34 taps, 24 rows per unit): more units than the tensor pipe stages
    pts.append((3240, 5760, ("opencv",), 384))
    for _, _, lo, hi in boundary_points():
        for side in (lo, hi):
            if side is not None:
                pts.append((side[1], side[2], ("opencv", "rgb"), 224))
    seen, out = set(), []
    for p in pts:
        key = (p[0], p[1], p[3])
        if key in seen:
            continue
        seen.add(key)
        out.append(p)
    return tuple(out)


def sweep_cases() -> list[tuple[int, int, str, int]]:
    """sweep() flattened to (width, height, fmt, res)."""
    return [(w, h, f, r) for w, h, fmts, r in sweep() for f in fmts]


# ------------------------------------------------------------------------------------------------ exact input classes
def constant_rgb(height: int, width: int, value) -> np.ndarray:
    """uint8 [H, W, 3] of one colour: the resize of a constant is that constant (the weights of an output sum to 1 within fp32 rounding,
    far inside the half LSB the u8 rounding allows)."""
    return np.broadcast_to(np.asarray(value, np.uint8), (height, width, 3)).copy()


def constant_nv12(height: int, width: int, y: int, u: int, v: int) -> np.ndarray:
    """uint8 [H * 3 / 2, W] NV12 of one colour; its RGB is color.nv12_to_rgb / nv12_to_rgb_swscale of it, one value per channel."""
    out = np.empty((height * 3 // 2, width), np.uint8)
    out[:height] = y
    out[height:, 0::2] = u
    out[height:, 1::2] = v
    return out


def constant_nv12_rgb(y: int, u: int, v: int, fmt: str) -> np.ndarray:
    """The one RGB colour of constant_nv12(y, u, v) in `fmt`'s arithmetic."""
    conv = color.nv12_to_rgb_swscale if fmt == "swscale" else color.nv12_to_rgb
    return conv(constant_nv12(2, 2, y, u, v), 2, 2)[0, 0]


# ------------------------------------------------------------------------------------------------ fast forms of the oracle chain
# The sweep runs the oracle at sources up to 6K.  These are color.nv12_to_rgb / nv12_to_rgb_swscale and preprocess.clip_resize_crop_u8
# restated on torch tensors, so that they can run on any device: integer colour arithmetic with the chroma terms at chroma resolution,
# and the resize as the same separate fp32 multiplies and adds in tap order (eager torch rounds each one, as numpy does), over the
# cropped outputs and the source rows they tap only.  tests/test_preprocess_plan_cpu.py checks them byte for byte against the numpy
# oracle.
def nv12_to_rgb_fast(nv12, height: int, width: int, fmt: str):
    """nv12: uint8 tensor [H * 3 / 2, >= W] -> uint8 tensor [H, W, 3]."""
    import torch

    y = nv12[:height, :width].to(torch.int32).reshape(height // 2, 2, width // 2, 2)
    uv = nv12[height : height + height // 2, :width].to(torch.int32)
    u, v = uv[:, 0::2][:, None, :, None], uv[:, 1::2][:, None, :, None]
    if fmt == "swscale":
        yy = (((y << 3) - color.SWS_YOFF) * color.SWS_Y) >> 16
        uu, vv = (u << 3) - color.SWS_COFF, (v << 3) - color.SWS_COFF
        planes = (yy + ((vv * color.SWS_VR) >> 16), yy + (((uu * color.SWS_UG) >> 16) + ((vv * color.SWS_VG) >> 16)), yy + ((uu * color.SWS_UB) >> 16))
    else:
        yy = torch.clamp(y - 16, min=0) * color.CY + (1 << (color.SHIFT - 1))
        u, v = u - 128, v - 128
        planes = ((yy + color.CVR * v) >> color.SHIFT, (yy + (color.CVG * v + color.CUG * u)) >> color.SHIFT, (yy + color.CUB * u) >> color.SHIFT)
    return torch.stack([q.reshape(height, width) for q in planes], dim=-1).clamp(0, 255).to(torch.uint8)


def _taps_last_axis(x, xmin, xsize, w):
    """preprocess._apply_taps_last_axis on a tensor: t = x0 * w0; t = t + xj * wj."""
    import torch

    idx = torch.from_numpy(np.minimum(xmin[:, None] + np.arange(w.shape[1])[None, :], x.shape[-1] - 1)).to(x.device)
    wt = torch.from_numpy(w).to(x.device)
    acc = x.index_select(-1, idx[:, 0]) * wt[:, 0]
    for t in range(1, w.shape[1]):
        acc = acc + x.index_select(-1, idx[:, t]) * wt[:, t]
    return acc


def resize_crop_u8_fast(frames_nhwc, res: int):
    """preprocess.clip_resize_crop_u8 on a tensor: uint8 [N, H, W, 3] -> uint8 [N, 3, res, res] on the same device."""
    import torch

    n, h, w, _ = frames_nhwc.shape
    new_w, new_h, top, left, tx, ty = cropped_taps(w, h, res)
    x = frames_nhwc.permute(0, 3, 1, 2)
    if (new_h, new_w) == (h, w):  # torchvision's early return
        return x[:, :, top : top + res, left : left + res].contiguous()
    x = x[:, :, ty[4] : ty[5], :].to(torch.float32)  # only the rows the cropped outputs tap
    x = _taps_last_axis(x, tx[0], tx[1], tx[2])
    x = _taps_last_axis(x.transpose(-1, -2).contiguous(), ty[0] - ty[4], ty[1], ty[2]).transpose(-1, -2)
    return torch.round(x.clamp(0, 255)).to(torch.uint8).contiguous()
