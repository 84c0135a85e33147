"""Times cb_gemm_f16 at the tower's GEMM shapes with CUDA events, each with the epilogue the tower gives it; optionally A/B against
a second build of libcurate_b200.so, the two timed alternately in one process.

    python tools/prof_gemm.py [--other path/to/libcurate_b200.so] [--seconds 1.0] [--rounds 3]

One JSON line per (shape, library): ms per launch (best round), TFLOP/s (2MNK) and algorithmic GB/s (A + W + output [+ residual
read], each once). torch.addmm (cuBLAS, fp16 out, no fused residual or activation) on the same shapes is printed as a same-card
yardstick, and the first line has the card name, power limit and max SM clock (nvidia-smi, read only).

Each library is loaded with RTLD_LOCAL and called through ctypes directly, so neither build's symbols can stand in for the other's.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
EPI_NONE, EPI_QUICK_GELU, EPI_GELU_TANH = 0, 1, 2
M_TOWER = 264 * 257  # the bench step: 264 frames x 257 tokens (CLIP ViT-L/14 at 224 px)

# name, M, N, K, output ("f16" / "f32"), epilogue, bias, in-place fp32 residual
SHAPES = [
    ("qkv", M_TOWER, 3072, 1024, "f16", EPI_NONE, True, False),
    ("out_proj", M_TOWER, 1024, 1024, "f32", EPI_NONE, True, True),
    ("fc1", M_TOWER, 4096, 1024, "f16", EPI_QUICK_GELU, True, False),
    ("fc2", M_TOWER, 1024, 4096, "f32", EPI_NONE, True, True),
    ("siglip_fc1", M_TOWER, 4304, 1152, "f16", EPI_GELU_TANH, True, False),
    ("patch_embed", 264 * 256, 1024, 640, "f32", EPI_NONE, False, False),
]


class Lib:
    def __init__(self, path: str, device: int):
        self.path = path
        self.so = C.CDLL(os.fspath(path), mode=C.RTLD_LOCAL)
        vp, i = C.c_void_p, C.c_int
        self.so.cb_init.restype, self.so.cb_init.argtypes = i, [i, C.POINTER(vp)]
        self.so.cb_last_error.restype, self.so.cb_last_error.argtypes = C.c_char_p, [vp]
        self.so.cb_gemm_f16.restype = i
        self.so.cb_gemm_f16.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, i, i, vp]
        self.h = vp()
        if self.so.cb_init(device, C.byref(self.h)) != 0:
            raise RuntimeError(f"cb_init failed for {path}")

    def gemm(self, a, w, bias, res, out, m, n, k, epi, stream):
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        o32, o16 = (ptr(out), None) if out.dtype == torch.float32 else (None, ptr(out))
        rc = self.so.cb_gemm_f16(self.h, ptr(a), ptr(w), ptr(bias), ptr(res), o32, o16, m, n, k, epi, stream)
        if rc != 0:
            raise RuntimeError(f"cb_gemm_f16 ({self.path}): {rc}: {self.so.cb_last_error(self.h).decode()}")


def card_info() -> dict:
    q = "name,power.limit,clocks.max.sm,clocks_event_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()  # fmt: skip
    except (OSError, subprocess.SubprocessError) as exc:
        out = f"nvidia-smi unavailable: {exc}"
    return {"card": out, "torch_name": torch.cuda.get_device_name()}


def time_fn(fn, seconds: float) -> float:
    """ms per call over a window of >= `seconds` (call count sized from a short probe)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        fn()
    e1.record()
    torch.cuda.synchronize()
    n = max(3, math.ceil(seconds * 1e3 / max(e0.elapsed_time(e1) / 3, 1e-3)))
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=str(ROOT / "cosmos_curate_b200" / "libcurate_b200.so"))
    ap.add_argument("--other", default=None, help="a second libcurate_b200.so to time alternately with --lib")
    ap.add_argument("--seconds", type=float, default=1.0, help="timed window per (shape, library, round)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_gemm: no CUDA device")
    dev = torch.cuda.current_device()
    print(json.dumps(card_info()), flush=True)
    libs = {"lib": Lib(args.lib, dev)}
    if args.other:
        libs["other"] = Lib(args.other, dev)
    stream = torch.cuda.current_stream().cuda_stream
    wanted = set(args.shapes.split(","))
    for name, m, n, k, odt, epi, has_bias, has_res in SHAPES:
        if name not in wanted:
            continue
        g = torch.Generator(device="cuda").manual_seed(m + n + k)
        a = (torch.randn(m, k, device="cuda", generator=g) * 0.5).half()
        w = (torch.randn(n, k, device="cuda", generator=g) * 0.05).half()
        bias = torch.randn(n, device="cuda", generator=g) if has_bias else None
        out = torch.empty(m, n, device="cuda", dtype=torch.float32 if odt == "f32" else torch.float16)
        if has_res:
            out.normal_(generator=g)
        res = out if has_res else None  # in place, as the tower runs it
        flop = 2.0 * m * n * k
        nbytes = m * k * 2 + n * k * 2 + m * n * out.element_size() + (m * n * 4 if has_res else 0)
        best = {key: float("inf") for key in libs}
        for lib in libs.values():  # warm-up: module load, tensor-map encode, clocks
            for _ in range(5):
                lib.gemm(a, w, bias, res, out, m, n, k, epi, stream)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for key, lib in libs.items():
                ms = time_fn(lambda: lib.gemm(a, w, bias, res, out, m, n, k, epi, stream), args.seconds)  # noqa: B023
                best[key] = min(best[key], ms)
        for key, ms in best.items():
            print(json.dumps({"shape": name, "lib": libs[key].path, "M": m, "N": n, "K": k, "out": odt, "residual": has_res, "ms": round(ms, 4),
                              "tflops": round(flop / ms / 1e9, 1), "gbs": round(nbytes / ms / 1e6, 1)}), flush=True)  # fmt: skip
        bh = bias.half() if bias is not None else torch.zeros(n, device="cuda", dtype=torch.float16)
        wt = w.t()
        ms = time_fn(lambda: torch.addmm(bh, a, wt), args.seconds)  # noqa: B023
        print(json.dumps({"shape": name, "lib": "torch.addmm (cuBLAS, fp16 out)", "M": m, "N": n, "K": k, "ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1)}),
              flush=True)  # fmt: skip
        del a, w, bias, out, res


if __name__ == "__main__":
    main()
