"""One-off GPU diagnostics: preprocess TMA variants + first NVDEC decode.  Usage: python tools/debug_gpu.py <what>"""
import ctypes as C
import sys

sys.path.insert(0, ".")
import numpy as np
import torch

from cosmos_curate_b200 import _lib
from cosmos_curate_b200.runtime import Context
from oracle import color, preprocess

what = sys.argv[1]
ctx = Context(0)
if what == "pre":
    for (h, w, pitch, lr) in ((64, 96, 128, 64), (1080, 1920, 2048, 1088)):
        f = color.synthetic_nv12(h, w, seed=1)
        buf = np.zeros((1, lr + h // 2, pitch), dtype=np.uint8)
        buf[0, :h, :w] = f[:h]
        buf[0, lr : lr + h // 2, :w] = f[h:]
        pool = ctx.nv12_pool(torch.from_numpy(buf).cuda(), w, h, lr)
        out = ctx.preprocess_clip_u8(pool).cpu().numpy()
        torch.cuda.synchronize()
        want = preprocess.clip_resize_crop_u8(color.nv12_to_rgb(f, h, w)[None], 224)
        d = np.abs(out.astype(int) - want.astype(int))
        print(f"{h}x{w}: maxdiff={d.max()} frac={(d>0).mean():.2e}", flush=True)
elif what == "dec":
    import cv2

    data = np.fromfile("tests/golden/sintel_clip_10s.mp4", dtype=np.uint8)
    lib = ctx.lib
    info = _lib.Mp4Info()
    pts = (C.c_int64 * 4096)()
    sync = (C.c_uint8 * 4096)()
    _lib.check(lib.cb_mp4_index(ctx.h, data.ctypes.data, data.size, C.byref(info), pts, sync, 4096), "cb_mp4_index", ctx.h)
    print("mp4:", info.codec, info.width, info.height, info.timescale, info.n_samples, info.n_sync, info.has_ctts, info.duration, list(pts[:5]))
    ids = np.array([0, 24, 48, 72, 96, 120, 144, 168, 192, 216, 239], dtype=np.int32)
    w, h = info.width, info.height
    pitch, lr = (w + 255) // 256 * 256, h
    buf = torch.zeros((len(ids), lr + h // 2, pitch), dtype=torch.uint8, device="cuda")
    pool = ctx.nv12_pool(buf, w, h, lr)
    dec = C.c_void_p()
    _lib.check(lib.cb_decoder_create(ctx.h, C.byref(dec)), "cb_decoder_create", ctx.h)
    stats = _lib.DecodeStats()
    slots = np.arange(len(ids), dtype=np.int32)
    import time

    for rep in range(3):
        t0 = time.time()
        _lib.check(lib.cb_decoder_decode(dec, data.ctypes.data, data.size, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids), C.byref(pool.desc),
                                         slots.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(stats)), "cb_decoder_decode", ctx.h)
        print(f"decode rep{rep}: {time.time()-t0:.3f}s decoded={stats.frames_decoded} emitted={stats.frames_emitted} coded={stats.coded_width}x{stats.coded_height} disp={stats.width}x{stats.height}")
    got = buf.cpu().numpy()
    cap = cv2.VideoCapture("tests/golden/sintel_clip_10s.mp4")
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    capc = cv2.VideoCapture("tests/golden/sintel_clip_10s.mp4")
    rgb = ctx.nv12_to_rgb(pool).cpu().numpy()
    k = 0
    for i in range(240):
        ok, y = cap.read()
        ok2, bgr = capc.read()
        if k < len(ids) and i == ids[k]:
            dy = np.abs(got[k, :h, :w].astype(int) - y.reshape(h, w).astype(int))
            drgb = np.abs(rgb[k].astype(int) - bgr[..., ::-1].astype(int))
            print(f"frame {i}: luma maxdiff={dy.max()}  rgb-vs-swscale maxdiff={drgb.max()} mean={drgb.mean():.3f}")
            k += 1
    lib.cb_decoder_destroy(dec)
