"""Times cb_attention_f16 at the bench shape (ViT-L/14: 264 images x 257 tokens, 16 heads x 64) with CUDA events; optionally A/B
against a second build of libcurate_b200.so, the two timed alternately in one process.

    python tools/prof_attn.py [--other path/to/libcurate_b200.so] [--n 264] [--seconds 1.0] [--rounds 3]

One JSON line per library: ms per launch (best round), TFLOP/s (4 T^2 d per head: QK^T and PV) and algorithmic GB/s (Q, K, V read
once, O written once).  With --other, a last line has the largest difference between the two builds' outputs on the same seeded
input.  The first line has the card name, power limit and max SM clock (nvidia-smi, read only).

Each library is loaded with RTLD_LOCAL and called through ctypes directly, so neither build's symbols can stand in for the other's.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tools.prof_gemm import card_info, time_fn  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
T, HEADS, HD = 257, 16, 64


class Lib:
    def __init__(self, path: str, device: int):
        self.path = path
        self.so = C.CDLL(os.fspath(path), mode=C.RTLD_LOCAL)
        vp, i = C.c_void_p, C.c_int
        self.so.cb_init.restype, self.so.cb_init.argtypes = i, [i, C.POINTER(vp)]
        self.so.cb_last_error.restype, self.so.cb_last_error.argtypes = C.c_char_p, [vp]
        self.so.cb_attention_f16.restype = i
        self.so.cb_attention_f16.argtypes = [vp, vp, vp, i, i, i, i, vp]
        self.h = vp()
        if self.so.cb_init(device, C.byref(self.h)) != 0:
            raise RuntimeError(f"cb_init failed for {path}")

    def attention(self, qkv, out, n, stream):
        rc = self.so.cb_attention_f16(self.h, qkv.data_ptr(), out.data_ptr(), n, T, HEADS, HD, stream)
        if rc != 0:
            raise RuntimeError(f"cb_attention_f16 ({self.path}): {rc}: {self.so.cb_last_error(self.h).decode()}")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=str(ROOT / "cosmos_curate_b200" / "libcurate_b200.so"))
    ap.add_argument("--other", default=None, help="a second libcurate_b200.so to time alternately with --lib")
    ap.add_argument("--n", type=int, default=264, help="images")
    ap.add_argument("--seconds", type=float, default=1.0, help="timed window per (library, round)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_attn: no CUDA device")
    dev = torch.cuda.current_device()
    print(json.dumps(card_info()), flush=True)
    libs = {"lib": Lib(args.lib, dev)}
    if args.other:
        libs["other"] = Lib(args.other, dev)
    stream = torch.cuda.current_stream().cuda_stream
    n, hidden = args.n, HEADS * HD
    g = torch.Generator(device="cuda").manual_seed(n)
    qkv = (torch.randn(n, T, 3 * hidden, device="cuda", generator=g) * 1.5).half()  # the tower's activation scale
    outs = {key: torch.empty(n, T, hidden, device="cuda", dtype=torch.float16) for key in libs}
    flop = 4.0 * n * HEADS * T * T * HD
    nbytes = n * T * (3 * hidden + hidden) * 2
    best = {key: float("inf") for key in libs}
    for key, lib in libs.items():  # warm-up: module load, tensor-map encode, clocks
        for _ in range(5):
            lib.attention(qkv, outs[key], n, stream)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for key, lib in libs.items():
            ms = time_fn(lambda: lib.attention(qkv, outs[key], n, stream), args.seconds)  # noqa: B023
            best[key] = min(best[key], ms)
    for key, ms in best.items():
        print(json.dumps({"lib": libs[key].path, "n": n, "T": T, "heads": HEADS, "head_dim": HD, "ms": round(ms, 4),
                          "tflops": round(flop / ms / 1e9, 1), "gbs": round(nbytes / ms / 1e6, 1)}), flush=True)  # fmt: skip
    if "other" in libs:
        a, b = outs["lib"].float(), outs["other"].float()
        diff = (a - b).abs()
        print(json.dumps({"max_abs_diff": diff.max().item(), "max_rel_diff": (diff / b.abs().clamp_min(1e-3)).max().item(),
                          "elements_differing": int((outs["lib"].view(torch.int16) != outs["other"].view(torch.int16)).sum())}), flush=True)  # fmt: skip


if __name__ == "__main__":
    main()
