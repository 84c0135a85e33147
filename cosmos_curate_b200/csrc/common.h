// Shared host-side declarations for libcurate_b200: context, error plumbing, TMA descriptor encode.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/curate_b200.h"

namespace cb {

void set_global_error(const char* msg);

struct TapTable {  // antialiased-bicubic tap table for one axis (device memory)
  int in_size = 0, out_size = 0, crop_off = 0, crop_len = 0, max_taps = 0;
  int src_begin = 0, src_end = 0;  // union of source indices touched by the cropped outputs
  int* d_min = nullptr;            // [crop_len] first source index per output
  int* d_size = nullptr;           // [crop_len] tap count per output
  float* d_w = nullptr;            // [crop_len * max_taps] normalised weights
  std::vector<int> h_min, h_size;
  std::vector<float> h_w;          // host copy of d_w (the tensor-pipe kernel builds its fp16 hi/lo operand tiles from it)
};

struct ResizeTaps {  // cv2.resize tap table for one axis (device memory): INTER_CUBIC (4 taps per output) or INTER_LINEAR (2)
  int* d_first = nullptr;    // [dst] source index of the first tap (unclamped)
  short* d_wq = nullptr;     // [dst][taps] weights quantised to 2^11 (OpenCV's own fixed-point path)
  double* d_wf = nullptr;    // [dst][4] unquantised cubic weights (IPP-style path, evaluated in double); null for linear
};

}  // namespace cb

struct cb_ctx {
  int device = 0;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  size_t total_mem = 0;
  std::string last_error;  // last failure on ANY thread (guarded by mu); cb_last_error() prefers the calling thread's own message
  std::mutex mu;
  PFN_cuTensorMapEncodeTiled_v12000 encode_tiled = nullptr;
  std::map<std::tuple<int, int, int, int>, cb::TapTable> taps;  // (in, out, crop_off, crop_len)
  std::map<std::tuple<int, int, int>, cb::ResizeTaps> resize_taps;  // (src, dst, TapKind in preprocess.cu)
  float* d_norm_lut = nullptr;                                  // [3*256] fp32, normalise LUT currently loaded
  float lut_mean[3] = {0, 0, 0}, lut_std[3] = {0, 0, 0};
  std::atomic<unsigned long long> launches{0};  // kernels launched by this library (bench.py reports it); decode threads launch too
  // per-category kernel timing (cb_profile_begin/end): one event before every launch, categories CB_PROF_*
  bool prof_on = false;
  std::vector<cudaEvent_t> prof_ev;
  std::vector<int> prof_cat;
  size_t prof_n = 0;
  void* nvdec = nullptr;            // lazily created NVDEC state (nvdec.cpp)
  uint8_t* d_tmp_u8 = nullptr;      // u8 [n][3][res][res] between a resample kernel and the normalise/pack kernel
  size_t tmp_u8_cap = 0;
  int* d_slots = nullptr;           // device staging of the slot list of the current preprocess call
  int slots_cap = 0;
};

namespace cb {

int fail(cb_ctx* ctx, int code, const char* fmt, ...);
// Called immediately before every kernel launch of the library: counts it and, when profiling, drops an event.
void mark_launch(cb_ctx* ctx, int category, cudaStream_t stream);

#define CB_CUDA(ctx, expr)                                                                                   \
  do {                                                                                                       \
    cudaError_t _e = (expr);                                                                                 \
    if (_e != cudaSuccess) return cb::fail(ctx, CB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// 2-D / 3-D tiled tensor map (row pitch etc. in BYTES); returns CB_OK or an error code.
int make_tensor_map(cb_ctx* ctx, CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* base, const uint64_t* dims,
                    const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box, CUtensorMapSwizzle swizzle);

const TapTable* get_taps(cb_ctx* ctx, int in_size, int out_size, int crop_off, int crop_len);
// The host half of get_taps: h_min, h_size, h_w, max_taps and the source range of one axis; allocates nothing.
void compute_taps(int in_size, int out_size, int crop_off, int crop_len, TapTable* t);
// preprocess_tc.cu: the tensor-pipe kernel's geometry for a request (host only, allocates nothing).  why is CB_PRE_WHY_OK when the kernel
// serves it, else the first limit it breaks (CB_PRE_WHY_KW, _RU, _UNITS, _SMEM).
struct TcGeometry {
  int nc = 0, n_slabs = 0, kw = 0, kb = 0, ru = 0, n_units = 0, y_begin = 0, why = 0;
  size_t smem = 0;
  std::vector<int> x_lo, k0, nk;  // [n_slabs] window start, [n_slabs * 2] first k-step and k-steps of each N-tile
};
void tc_geometry(const TapTable& tx, const TapTable& ty, int res, TcGeometry* g);
// preprocess_tc.cu: tensor-pipe resample into u8 [n][3][res][res] (returns CB_OK, 1 = configuration not served -> use the SIMT kernel,
// < 0 = error)
int run_clip_preprocess_tc(cb_ctx* ctx, const cb_surface_pool* pool, const int* d_slots, int n, int max_slot, int res, const TapTable* tx,
                           const TapTable* ty, uint8_t* out, cudaStream_t stream);
void release_tc_plans(cb_ctx* ctx);
int ensure_norm_lut(cb_ctx* ctx, const float mean[3], const float std_[3], cudaStream_t stream);
// NV12 -> RGB -> bilinear out_w x out_h for ONE surface at `base` (used on NVDEC-mapped frames), u8 HWC into `out`.
int bilinear_from_surface(cb_ctx* ctx, const void* base, int pitch, int luma_rows, int w, int h, int out_w, int out_h, uint8_t* out, cudaStream_t stream);
int run_clip_preprocess(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int res, int out_mode, int layout_patch,
                        int k_pad, int dtype, const float mean[3], const float std_[3], void* out, cudaStream_t stream);
// cb_video_tube's resize + normalise of n frames of `pool` to size x size, written as the video tower's fp16 patch rows
// [n][(size / patch)^2][k_pad] (pad columns zeroed).  n == 0 is a no-op.
int video_tube_patches(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int size, int patch, int k_pad, const float mean[3],
                       const float std_[3], void* out_f16, cudaStream_t stream);

// Tower ops (gemm.cu, vit_kernels.cu, attention_*.cu): fp16 operands, fp32 accumulation, launched on `stream`.
int gemm_f16(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* residual, float* out_f32, void* out_f16, int M,
             int N, int K, int epilogue, cudaStream_t stream);
int gemm_f16_ex(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* gamma, const float* residual, float* out_f32,
                void* out_f16, int M, int N, int K, int epilogue, cudaStream_t stream);
int layernorm_f16(cb_ctx* ctx, const float* x, const float* gamma, const float* beta, void* y, int rows, int d, float eps, cudaStream_t stream);
int layernorm_post_f16(cb_ctx* ctx, float* h, const float* gamma, const float* beta, void* y, int rows, int d, float eps, cudaStream_t stream);
int rmsnorm_f16(cb_ctx* ctx, const float* x, const float* w, void* y, int rows, int d, float eps, cudaStream_t stream);
int qk_rmsnorm_f16(cb_ctx* ctx, void* qkv, const float* wq, const float* wk, int rows, int d, float eps, cudaStream_t stream);
int assemble_tokens(cb_ctx* ctx, const float* patch, const float* cls, const float* pos, const float* gamma, const float* beta, float* h, int n,
                    int tokens, int grid2, int d, float eps, cudaStream_t stream);
int attention_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream);
int attention_wgmma(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream, bool* launched);
int attention_masked_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, const int* lengths, cudaStream_t stream);
int attention_stream_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream);
int map_pool(cb_ctx* ctx, const void* kv, const float* q, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream);
int clip_tail(cb_ctx* ctx, const float* h, size_t img_stride, const float* gamma, const float* beta, const float* proj, int d, int proj_dim,
              float eps, const float* aes_w, float aes_b, float* emb_out, float* feat_out, float* score_out, int n, cudaStream_t stream);
int l2norm_score(cb_ctx* ctx, const float* feat, int d, const float* aes_w, float aes_b, float* emb, float* feat_out, float* score, int n,
                 cudaStream_t stream);
int tube_patches(cb_ctx* ctx, const float* tubes, void* out, int frames, int image_size, int patch, int k_pad, cudaStream_t stream);
int token_mean(cb_ctx* ctx, const float* h, float* out, int n, int tokens, int d, cudaStream_t stream);
int clip_pool(cb_ctx* ctx, const float* q, const void* k, const void* v, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream);

}  // namespace cb
