// NV12 -> RGB colour arithmetic, the one definition every preprocess kernel uses.  Each arithmetic is split the way the
// block-structured kernels use it: a luma term per Y sample, three chroma terms per (U, V) pair, and a clamp-and-combine step
// (add-min-relu, DPX) per channel.
#pragma once
#include "common.h"

namespace cb {

// OpenCV ITUR_BT_601 fixed point (shift 20): cvtColor / CV-CUDA NV12 -> RGB.  The clamp before the shift equals min/max after it.
struct ColourOpenCv {
  static __device__ __forceinline__ int luma(int y) { return max(y - 16, 0) * 1220542 + (1 << 19); }
  static __device__ __forceinline__ void chroma(int u, int v, int& r, int& g, int& b) {
    u -= 128;
    v -= 128;
    r = 1673527 * v, g = -852492 * v - 409993 * u, b = 2116026 * u;
  }
  static __device__ __forceinline__ int combine(int luma, int chroma) { return __viaddmin_s32_relu(luma, chroma, (256 << 20) - 1) >> 20; }
};

// libswscale's unscaled yuv420p -> rgb24 converter (x86 SIMD path, libswscale/x86/yuv_2_rgb.asm; coefficients from
// ff_yuv2rgb_c_init_tables for ITU-R BT.601 limited range, the default PyAV / cv2 leave in place): 16-bit fixed point,
// every product truncated by pmulhw - (8Y - 128) * 9539 >> 16 etc. - nearest chroma.  This is what the reference's CPU decode
// (decode_video_cpu_frame_ids -> frame.to_ndarray(format="rgb24"), decoder_utils.py:439-451) feeds the CLIP transforms.
// Pinned bit-exactly against cv2/libswscale over the whole u8 range (tests/test_oracle_cpu.py).
struct ColourSws {
  static __device__ __forceinline__ int luma(int y) { return (((y << 3) - 128) * 9539) >> 16; }
  static __device__ __forceinline__ void chroma(int u, int v, int& r, int& g, int& b) {
    const int uu = (u << 3) - 1024, vv = (v << 3) - 1024;
    r = (vv * 13075) >> 16, g = ((uu * -3209) >> 16) + ((vv * -6660) >> 16), b = (uu * 16525) >> 16;
  }
  static __device__ __forceinline__ int combine(int luma, int chroma) { return __viaddmin_s32_relu(luma, chroma, 255); }
};

template <class C>
__device__ __forceinline__ void yuv_to_rgb(int y, int u, int v, int& r, int& g, int& b) {
  int cr, cg, cb_;
  C::chroma(u, v, cr, cg, cb_);
  const int l = C::luma(y);
  r = C::combine(l, cr), g = C::combine(l, cg), b = C::combine(l, cb_);
}

}  // namespace cb
