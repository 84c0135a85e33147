"""Host H.264 / HEVC decode for devices whose NVDEC is not usable from the process (runtime.nvdec_available), with the
libavformat / libavcodec that OpenCV has loaded: cv2.VideoCapture itself returns the luma plane only, the surface pools need NV12.
Decoding is normative, so the pictures are NVDEC's bit for bit.  Four struct fields are read at fixed offsets
(AVFormatContext.streams, AVStream.codecpar, AVPacket.stream_index, leading AVFrame fields); they hold for the library majors
listed in _MAJORS (FFmpeg 5 to 8), and any other version is refused at load."""

from __future__ import annotations

import ctypes as C
import os

import numpy as np

_libs = None
_MAJORS = {"libavformat": (59, 62), "libavcodec": (59, 62), "libavutil": (57, 60)}  # FFmpeg 5.0 .. 8.0


def _load():
    global _libs
    if _libs is None:
        import cv2  # noqa: F401 - loads its bundled libav* into the process

        paths = {}
        with open("/proc/self/maps") as f:
            for line in f:
                p = line.split()[-1]
                for name in ("libavformat", "libavcodec", "libavutil"):
                    if os.path.basename(p).startswith(name):
                        paths[name] = p
        if len(paths) != 3:
            raise RuntimeError("host decode needs the libavformat / libavcodec / libavutil that OpenCV loads; not found in this process")
        fmt, cod, utl = (C.CDLL(paths[n]) for n in ("libavformat", "libavcodec", "libavutil"))
        for name, lib, fn in (("libavformat", fmt, "avformat_version"), ("libavcodec", cod, "avcodec_version"), ("libavutil", utl, "avutil_version")):
            major, (lo, hi) = getattr(lib, fn)() >> 16, _MAJORS[name]
            if not lo <= major <= hi:
                raise RuntimeError(f"host decode: {name} major {major} is outside the supported {lo}..{hi} (struct offsets unverified)")
        P, I = C.c_void_p, C.c_int
        fmt.avformat_open_input.argtypes, fmt.avformat_open_input.restype = [C.POINTER(P), C.c_char_p, P, P], I
        fmt.avformat_find_stream_info.argtypes, fmt.avformat_find_stream_info.restype = [P, P], I
        fmt.av_find_best_stream.argtypes, fmt.av_find_best_stream.restype = [P, I, I, I, C.POINTER(P), I], I
        fmt.av_read_frame.argtypes, fmt.av_read_frame.restype = [P, P], I
        fmt.avformat_close_input.argtypes = [C.POINTER(P)]
        cod.avcodec_alloc_context3.argtypes, cod.avcodec_alloc_context3.restype = [P], P
        cod.avcodec_parameters_to_context.argtypes, cod.avcodec_parameters_to_context.restype = [P, P], I
        cod.avcodec_open2.argtypes, cod.avcodec_open2.restype = [P, P, P], I
        cod.avcodec_send_packet.argtypes, cod.avcodec_send_packet.restype = [P, P], I
        cod.avcodec_receive_frame.argtypes, cod.avcodec_receive_frame.restype = [P, P], I
        cod.avcodec_flush_buffers.argtypes = [P]
        cod.avcodec_free_context.argtypes = [C.POINTER(P)]
        cod.av_packet_alloc.restype = P
        cod.av_packet_unref.argtypes = [P]
        cod.av_packet_free.argtypes = [C.POINTER(P)]
        utl.av_frame_alloc.restype = P
        utl.av_frame_unref.argtypes = [P]
        utl.av_frame_free.argtypes = [C.POINTER(P)]
        _libs = (fmt, cod, utl)
    return _libs


class _Frame(C.Structure):  # leading fields of AVFrame
    _fields_ = [("data", C.c_void_p * 8), ("linesize", C.c_int * 8), ("extended_data", C.c_void_p), ("width", C.c_int), ("height", C.c_int),
                ("nb_samples", C.c_int), ("format", C.c_int)]  # fmt: skip


_YUV420P, _YUVJ420P = 0, 12
_EAGAIN, _EOF = -11, -541478725


def _plane(ptr: int, stride: int, rows: int, cols: int) -> np.ndarray:
    a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(rows * stride,))
    return a.reshape(rows, stride)[:, :cols]


def decode(data: np.ndarray, sync: np.ndarray, runs: list[tuple[int, int]], on_frame) -> tuple[int, int, int]:
    """Decode the mp4 in `data`.  `runs` = [(first sample, last display index wanted)] per stretch to decode, each starting at a sync
    sample (sample order = decode order; `sync` flags per sample); samples outside the runs are not decoded.  Calls
    on_frame(display index, y, u, v) with views valid during the call, for every picture of a run up to its last wanted index.
    Returns (pictures decoded, width, height).  Raises ValueError on a stream this path does not handle."""
    fmt, cod, utl = _load()
    fd = os.memfd_create("cb_clip")
    try:
        os.write(fd, memoryview(np.ascontiguousarray(data)))
        ctx, dec = C.c_void_p(), C.c_void_p()
        if fmt.avformat_open_input(C.byref(ctx), f"/proc/self/fd/{fd}".encode(), None, None) < 0:
            raise ValueError("libavformat cannot open the clip")
        pkt, frm, cc = cod.av_packet_alloc(), utl.av_frame_alloc(), C.c_void_p()
        try:
            if fmt.avformat_find_stream_info(ctx, None) < 0:
                raise ValueError("no stream info")
            vs = fmt.av_find_best_stream(ctx, 0, -1, -1, C.byref(dec), 0)  # AVMEDIA_TYPE_VIDEO
            if vs < 0 or not dec:
                raise ValueError("no decodable video stream")
            streams = C.cast(ctx.value + 48, C.POINTER(C.POINTER(C.c_void_p)))[0]  # AVFormatContext.streams
            codecpar = C.cast(streams[vs] + 16, C.POINTER(C.c_void_p))[0]  # AVStream.codecpar
            cc = C.c_void_p(cod.avcodec_alloc_context3(dec))
            if cod.avcodec_parameters_to_context(cc, codecpar) < 0 or cod.avcodec_open2(cc, dec, None) < 0:
                raise ValueError("libavcodec cannot open the decoder")
            f = C.cast(frm, C.POINTER(_Frame)).contents
            decoded = width = height = 0
            run_of = {}
            for first, last in runs:
                run_of[first] = last
            sample, active, disp, last, done = -1, False, 0, -1, False

            def drain() -> bool:
                nonlocal decoded, disp, width, height
                while disp <= last:
                    rc = cod.avcodec_receive_frame(cc, frm)
                    if rc in (_EAGAIN, _EOF):
                        return rc == _EOF
                    if rc < 0:
                        raise ValueError(f"avcodec_receive_frame failed ({rc})")
                    if f.format not in (_YUV420P, _YUVJ420P):
                        raise ValueError("only 8-bit 4:2:0 streams are supported")
                    width, height = f.width, f.height
                    decoded += 1
                    ch, cw = (height + 1) // 2, (width + 1) // 2
                    on_frame(disp, _plane(f.data[0], f.linesize[0], height, width), _plane(f.data[1], f.linesize[1], ch, cw), _plane(f.data[2], f.linesize[2], ch, cw))
                    utl.av_frame_unref(frm)
                    disp += 1
                return False

            while not done and fmt.av_read_frame(ctx, pkt) >= 0:
                if C.cast(pkt + 36, C.POINTER(C.c_int))[0] != vs:  # AVPacket.stream_index
                    cod.av_packet_unref(pkt)
                    continue
                sample += 1
                if sample in run_of:  # a run starts here: pictures of earlier stretches are complete or unwanted
                    if active:
                        cod.avcodec_send_packet(cc, None)
                        drain()
                    cod.avcodec_flush_buffers(cc)
                    active, disp, last = True, sample, run_of[sample]
                elif active and sync[sample] and disp > last:
                    active = False
                if active and disp <= last:
                    if cod.avcodec_send_packet(cc, pkt) < 0:
                        cod.av_packet_unref(pkt)
                        raise ValueError("avcodec_send_packet failed")
                    drain()
                    if disp > last and sample >= max(run_of):
                        done = True
                cod.av_packet_unref(pkt)
            if active and disp <= last:
                cod.avcodec_send_packet(cc, None)
                drain()
            return decoded, width, height
        finally:
            if cc:
                cod.avcodec_free_context(C.byref(cc))
            p, q = C.c_void_p(pkt), C.c_void_p(frm)
            cod.av_packet_free(C.byref(p))
            utl.av_frame_free(C.byref(q))
            fmt.avformat_close_input(C.byref(ctx))
    finally:
        os.close(fd)
