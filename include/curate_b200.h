/* libcurate_b200 - C ABI of the B200-native decode -> sample -> preprocess -> embed/classify path.
 *
 * The reference (nvidia-cosmos/cosmos-curate) has NO FFI boundary on this path: its stages call
 * Python libraries (PyAV, PyNvVideoCodec, CV-CUDA, torchvision, transformers).  The drop-in boundary
 * is therefore the Python plugin surface (CuratorStage / ModelInterface, mirrored in
 * cosmos_curate_b200/); this header is the thin C ABI those Python stages bind with ctypes.  Every entry
 * point names the reference call it replaces (file:line relative to the reference checkout).
 *
 * Conventions: plain pointers and sizes only (no torch types); every function returns CB_OK (0) or a
 * negative error code and never throws; cb_last_error() returns the message.  Device pointers are
 * caller-owned (torch-allocated is fine); the library owns only its context, cached tables, model
 * weights/workspace and NVDEC sessions.  `stream` is a cudaStream_t passed as void* (NULL = default).
 * There is no CPU fallback anywhere: without a CUDA device cb_init fails.
 */
#ifndef CURATE_B200_H
#define CURATE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CB_OK 0
#define CB_ERR_CUDA (-1)        /* CUDA runtime / driver error */
#define CB_ERR_ARG (-2)         /* bad argument */
#define CB_ERR_UNSUPPORTED (-3) /* valid request this build cannot serve (size, codec, ...) */
#define CB_ERR_NVDEC (-4)       /* libnvcuvid missing or decode failure */
#define CB_ERR_DEMUX (-5)       /* malformed / unsupported container */
#define CB_ERR_STATE (-6)       /* call order (e.g. forward before finalize) */
#define CB_ERR_INVALID (-7)     /* input data out of range (e.g. a token id >= vocab, a text length outside [1, L]) */

#define CB_ABI_VERSION 1

typedef struct cb_ctx cb_ctx;
typedef struct cb_vit cb_vit;

/* ---- context ------------------------------------------------------------------------------------ */
int cb_abi_version(void);
/* Creates a context on CUDA device `device` (must be sm_90).  Replaces the implicit torch/CV-CUDA
 * device setup of nvcodec_utils.py:337 (device_id hard-coded to 0 there) and clip.py:39. */
int cb_init(int device, cb_ctx** out);
void cb_destroy(cb_ctx* ctx);
/* Message of the last failing call on `ctx` (or of the last failing cb_init when ctx == NULL). */
const char* cb_last_error(cb_ctx* ctx);
int cb_device_info(cb_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem);
/* PCI bus id of the context's device ("0000:1b:00.0") into buf[len]: the host side uses it to find the GPU's NUMA node
 * (/sys/bus/pci/devices/<id>/numa_node) and pin the NVDEC feeder threads next to it.  The reference leaves placement to
 * Ray/xenna (cosmos-xenna resources.py); one process per GPU needs it spelled out. */
int cb_device_pci_bus_id(cb_ctx* ctx, char* buf, int len);
/* Number of kernels this library has launched on `ctx` since cb_init (bench.py "gpu_launches"). */
unsigned long long cb_launch_count(cb_ctx* ctx);

/* Per-kernel-category device timing: an event is recorded before every launch between begin and end; end
 * returns the summed milliseconds and launch counts per category (bench.py's roofline figures). */
#define CB_PROF_PREPROCESS 0
#define CB_PROF_GEMM 1
#define CB_PROF_LAYERNORM 2
#define CB_PROF_ATTENTION 3
#define CB_PROF_OTHER 4
#define CB_PROF_CONV 5 /* shot-detection network (cb_transnet_*) */
#define CB_PROF_CATEGORIES 6
int cb_profile_begin(cb_ctx* ctx);
int cb_profile_end(cb_ctx* ctx, void* stream, float* ms_by_category, int* launches_by_category, int n_categories);

/* ---- surfaces ----------------------------------------------------------------------------------- */
#define CB_FMT_NV12 0  /* Y plane [luma_rows x pitch] then interleaved UV plane [height/2 x pitch] */
#define CB_FMT_RGB24 1 /* interleaved RGB u8, pitch >= 3*width */
/* NV12 surfaces (same layout as CB_FMT_NV12) whose colour conversion follows libswscale's unscaled yuv420p -> rgb24 converter
 * bit for bit - what the reference's CPU decode hands to CLIP (frame.to_ndarray(format="rgb24"), decoder_utils.py:439-451).
 * CB_FMT_NV12 converts with OpenCV / CV-CUDA semantics (cvcuda.cvtcolor_into, nvcodec_utils.py:35-38,178), the reference's
 * CUDA branch (27x48 shot-detection frames).  Both: ITU-R BT.601 limited range, nearest chroma. */
#define CB_FMT_NV12_SWS 2

/* A pool of equally shaped frames in device memory: frame i starts at base + i*slot_stride.
 * NV12: UV plane of a frame starts `luma_rows * pitch` bytes after its Y plane (NVDEC aligns the coded
 * height, so luma_rows >= height).  base, pitch and slot_stride must be multiples of 16 bytes. */
typedef struct cb_surface_pool {
  const void* base;
  size_t slot_stride;
  int width, height; /* display size in pixels */
  int pitch;         /* bytes per row */
  int luma_rows;     /* NV12 only: rows between the Y plane and the UV plane */
  int format;        /* CB_FMT_* */
} cb_surface_pool;

/* ---- preprocess ---------------------------------------------------------------------------------- */
#define CB_DT_F16 0
#define CB_DT_BF16 1
#define CB_DT_F32 2
#define CB_LAYOUT_NCHW 0  /* out[n][3][res][res]                                   (reference tensor layout) */
#define CB_LAYOUT_PATCH 1 /* out[n][(res/patch)^2][k_pad], k = (c, py, px), zero padded (tower input) */

/* Colour-convert + resize + crop + normalise + pack.  Replaces cvcuda.cvtcolor_into (nvcodec_utils.py:178)
 * and the reference CLIP transform chain Resize(res, bicubic, antialias) -> CenterCrop(res) -> /255 ->
 * Normalize (clip.py:48-62) with one pass over the source frame (colour, resize, crop -> u8 image) and
 * one pass over the u8 image (normalise, pack).
 * slots[n] (host) selects the frames of `pool`; `out` is device memory of the chosen layout/dtype. */
int cb_preprocess_clip(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int res, int layout, int patch,
                       int k_pad, int dtype, const float mean[3], const float std_[3], void* out, void* stream);

/* The same resize/crop with the u8 stage exposed: out u8 [n][3][res][res] (parity tests; this is the
 * tensor torchvision produces before ConvertImageDtype, clip.py:50-55). */
int cb_preprocess_clip_u8(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int res, uint8_t* out,
                          void* stream);

/* Which resample kernel cb_preprocess_clip / cb_preprocess_clip_u8 would run for a width x height pool of `format` at `res`, and
 * its geometry.  Launches nothing, allocates nothing and reads no environment; ctx may be null (then errors carry no message).
 * Returns CB_ERR_ARG for a null `out`, an unknown format, a size <= 0 or res outside 1..1024, else CB_OK with `out` filled: a
 * request the library refuses with CB_ERR_UNSUPPORTED (odd NV12 size, more than 64 taps on an axis) has kernel = CB_PRE_NONE. */
#define CB_PRE_NONE 0 /* the call returns CB_ERR_UNSUPPORTED */
#define CB_PRE_TC 1   /* clip_preprocess_tc_kernel: horizontal pass on the tensor pipe (NV12 only) */
#define CB_PRE_SIMT 2 /* clip_preprocess_simt_kernel */
/* why a kernel does not serve a request (tc_why, simt_why) */
#define CB_PRE_WHY_OK 0
#define CB_PRE_WHY_RGB 1    /* tensor pipe: RGB pools */
#define CB_PRE_WHY_TAPS40 2 /* tensor pipe: more than 40 vertical taps */
#define CB_PRE_WHY_KW 3     /* tensor pipe: a 16-column slab's source window exceeds one 256-byte TMA box */
#define CB_PRE_WHY_RU 4     /* tensor pipe: fewer than 16 source rows per unit */
#define CB_PRE_WHY_UNITS 5  /* tensor pipe: more units per frame column than the kernel stages */
#define CB_PRE_WHY_SMEM 6   /* more than 227 KB of shared memory */
#define CB_PRE_WHY_TAPS64 7 /* more than 64 taps on either axis: neither kernel */
#define CB_PRE_WHY_SWA 8    /* SIMT: an 8-column tile's source window exceeds one 256-byte TMA box */
#define CB_PRE_WHY_ODD 9    /* NV12 with an odd width or height: neither kernel */
typedef struct cb_preprocess_plan_info {
  int kernel;          /* CB_PRE_*: what the default call runs */
  int simt_kernel;     /* what the call runs with CB_PRE_KERNEL=simt: CB_PRE_SIMT or CB_PRE_NONE */
  int tc_why, simt_why;                /* CB_PRE_WHY_* of each kernel */
  int new_w, new_h, top, left;         /* Resize(res) output size (short side -> res) and CenterCrop(res) offsets */
  int taps_x, taps_y;                  /* widest tap window of the cropped outputs per axis */
  int src_y_begin, src_y_end;          /* source rows the cropped outputs tap */
  /* tensor-pipe geometry; zero when taps_x or taps_y > 64 or the request is refused */
  int tc_nc, tc_n_slabs, tc_kw, tc_kb, tc_ru, tc_n_units, tc_y_begin, tc_smem;
  /* SIMT geometry; zero when taps_x or taps_y > 64 or the request is refused */
  int simt_tc, simt_tiles, simt_swa, simt_gu, simt_ring, simt_n_strips, simt_y_begin, simt_smem;
} cb_preprocess_plan_info;
int cb_preprocess_plan(cb_ctx* ctx, int width, int height, int format, int res, cb_preprocess_plan_info* out);

/* Fused NV12->RGB + bilinear resize to out_w x out_h, u8 HWC: out[n][out_h][out_w][3].  Replaces
 * cvcuda.cvtcolor_into + cvcuda.resize_into(Interp.LINEAR) (nvcodec_utils.py:178,189-194), the
 * 27x48 shot-detection frames of VideoFrameExtractionStage (frame_extraction_stages.py:112-116). */
int cb_preprocess_bilinear_u8(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int out_w, int out_h,
                              uint8_t* out, void* stream);

#define CB_CUBIC_OPENCV 0 /* OpenCV's own fixed-point code: aarch64 wheels, x86 wheels with IPP disabled - bit-exact */
#define CB_CUBIC_IPP 1    /* x86 opencv-python wheels dispatch to Intel IPP: correctly rounded float cubic (<= 1 LSB on ~1e-5 of pixels) */
/* cv2.resize(frame, (out_w, out_h), interpolation=cv2.INTER_CUBIC) of the RGB image of every selected frame (NV12 surfaces
 * are colour-converted per tap), u8 HWC out[n][out_h][out_w][3].  The optional `target_res` square resize of extract_frames
 * (decoder_utils.py:666-670; clip_extraction_target_res = 224 in benchmarks/split_pipeline/invoke.json:38): Keys cubic
 * a = -0.75, 4 taps per axis at any scale (no antialiasing, aspect ratio not preserved), border replicate. */
int cb_resize_cubic_u8(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int out_w, int out_h, int mode,
                       uint8_t* out, void* stream);

/* The video embedding towers' input formulation, per selected frame: cv2.resize(frame, (out_w, out_h)) [INTER_LINEAR on
 * uint8: OpenCV's fixed-point arithmetic bit for bit, incl. its INTER_AREA reroute of an exact 2x2 decimation] then
 * ((x / 255 - mean) / std) in float32.  Replaces InternVideo2MultiModality._construct_frames / _normalize
 * (cosmos_curate/models/internvideo2_mm.py:385-405), called by InternVideo2FrameCreationStage
 * (pipelines/video/embedding/internvideo2_stages.py:177).  RGB or NV12 pools (NV12 is colour-converted per tap).
 * out_f32 [n][3][out_h][out_w] and/or out_u8 [n][out_h][out_w][3] (the resized frames before normalisation); either may be
 * null, not both. */
int cb_video_tube(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int out_w, int out_h, const float mean[3],
                  const float std_[3], float* out_f32, uint8_t* out_u8, void* stream);
/* cb_video_tube at size x size written straight as the InternVideo2 tower's patch rows: out_f16 [n][(size / patch)^2][k_pad], k = (c, y, x)
 * of the patch, columns 3 patch^2 .. k_pad - 1 written as zeros.  Each value is the fp16 rounding (round to nearest even) of the fp32
 * value cb_video_tube gives, so this equals cb_tube_patches(cb_video_tube(...)) bit for bit.  Replaces _construct_frames
 * (models/internvideo2_mm.py:390-405) and the PatchEmbed input of the tower (internvideo2.py PatchEmbed, the Conv3d's im2col) in one
 * launch.  k_pad even and >= 3 patch^2, size >= patch; n == 0 is a no-op. */
int cb_video_tube_patches(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, int size, int patch, int k_pad, const float mean[3],
                          const float std_[3], void* out_f16, void* stream);

/* Full-resolution NV12 -> RGB24 (HWC, tightly packed): what decode_video_cpu_frame_ids returns per
 * frame (decoder_utils.py:439-451) / cvcuda.cvtcolor_into (nvcodec_utils.py:178).  Only for callers that
 * must hand RGB frames to an unmodified downstream stage. */
int cb_nv12_to_rgb(cb_ctx* ctx, const cb_surface_pool* pool, const int32_t* slots, int n, uint8_t* out, void* stream);

/* ---- image tower (CLIP / SigLIP style ViT) + aesthetic head --------------------------------------- */
#define CB_ACT_QUICK_GELU 0
#define CB_ACT_GELU_TANH 1
#define CB_ARCH_CLIP 0   /* CLS token, pre-LN, post-LN on CLS, bias-free projection (HF CLIPVisionModel) */
#define CB_ARCH_SIGLIP 1 /* no CLS, patch bias, post-LN on all tokens, MAP pooling head (HF SiglipVisionModel) */

typedef struct cb_vit_cfg {
  int image_size, patch, hidden, layers, heads, mlp, proj_dim;
  int act;  /* CB_ACT_* */
  int arch; /* CB_ARCH_* */
  float ln_eps;
} cb_vit_cfg;

/* Replaces CLIPModel.from_pretrained(...).to(device) (clip.py:41) for the image tower. */
int cb_vit_create(cb_ctx* ctx, const cb_vit_cfg* cfg, cb_vit** out);
void cb_vit_destroy(cb_vit* vit);
/* Upload one named tensor (host fp32, row-major, `count` elements).  Names: patch_w[hidden][3*p*p],
 * patch_b, cls, pos[tokens][hidden], pre_ln_w/b, L<i>.{ln1_w,ln1_b,qkv_w[3h][h],qkv_b,out_w,out_b,ln2_w,
 * ln2_b,fc1_w[mlp][h],fc1_b,fc2_w[h][mlp],fc2_b}, post_ln_w/b, proj_w[proj][hidden], map_* (SigLIP).
 * Tower handle lifecycle (cb_vit, cb_iv2, cb_iv2_text): set_tensor every tensor, then finalize, then forward.  A set_tensor call
 * (replacing a tensor included) un-finalizes the handle: forward returns CB_ERR_STATE until the next finalize, which also re-derives
 * what it folds from the weights (SigLIP's pooling query).  cb_vit_set_aesthetic writes in place and needs no new finalize. */
int cb_vit_set_tensor(cb_vit* vit, const char* name, const float* data, size_t count);
/* Aesthetic head folded to score = w . embedding + b (the reference MLP, aesthetics.py:44-53, has no
 * non-linearity).  w has proj_dim (or hidden) entries.  Optional. */
int cb_vit_set_aesthetic(cb_vit* vit, const float* w, size_t count, float b);
/* Checks that every tensor arrived and sizes the workspace for batches up to max_batch images. */
int cb_vit_finalize(cb_vit* vit, int max_batch);
/* K padding (in fp16 elements) the tower expects of CB_LAYOUT_PATCH input rows. */
int cb_vit_k_pad(const cb_vit* vit);
/* Forward over n preprocessed images.  patches: device fp16 [n][(image/patch)^2][k_pad] (CB_LAYOUT_PATCH).
 * emb_out: device fp32 [n][proj_dim or hidden], L2-normalised (clip.py:71-74).  feat_out (nullable):
 * the un-normalised features.  score_out (nullable): device fp32 [n] aesthetic scores
 * (clip_aesthetics.py:63-76). */
int cb_vit_forward(cb_vit* vit, const void* patches, int n, float* emb_out, float* feat_out, float* score_out, void* stream);
/* Preprocess + forward in one call: frames of `pool` -> embeddings / scores (the whole
 * CLIPAestheticScorer.__call__, clip_aesthetics.py:63-76, from NV12 or RGB frames). */
int cb_vit_embed_surfaces(cb_vit* vit, const cb_surface_pool* pool, const int32_t* slots, int n, const float mean[3],
                          const float std_[3], float* emb_out, float* feat_out, float* score_out, void* stream);

/* score[i] = w . emb[i] + b over device fp32 embeddings [n][d] (w: device fp32 [d]).  The reference's
 * AestheticScorer.__call__ (aesthetics.py:94-106) on already-computed embeddings. */
int cb_affine_score(cb_ctx* ctx, const float* emb, const float* w, float b, float* out, int n, int d, void* stream);

/* ---- demux + NVDEC ---------------------------------------------------------------------------- */
typedef struct cb_decoder cb_decoder;

typedef struct cb_mp4_info {
  int codec;          /* 4 = H.264, 8 = HEVC (cudaVideoCodec numbering) */
  int width, height;  /* sample-entry (display) size */
  uint32_t timescale; /* mdhd timescale: PTS seconds = pts / timescale */
  int n_samples, n_sync, has_ctts;
  uint64_t duration;     /* mdhd duration in `timescale` ticks */
  uint64_t sample_bytes; /* sum of the video sample sizes (stream bit rate = 8 * sample_bytes / seconds) */
} cb_mp4_info;

typedef struct cb_decode_stats {
  int frames_decoded, frames_emitted;
  int coded_width, coded_height, width, height;
} cb_decode_stats;

/* Index the first video track of an in-memory MP4: per-sample composition timestamps (decode order, in
 * `timescale` ticks, edit list applied) and sync flags.  Replaces the container open + packet demux of
 * get_video_timestamps (decoder_utils.py:230-278); the caller sorts and converts to float32 seconds exactly
 * as the reference does.  pts_out / sync_out (nullable) receive min(cap, n_samples) entries.  Host-only: ctx may
 * be NULL. */
int cb_mp4_index(cb_ctx* ctx, const uint8_t* data, size_t size, cb_mp4_info* info, int64_t* pts_out, uint8_t* sync_out, int cap);

/* Stream-copy cut (no transcode): samples [first_sample, first_sample + n_samples) of the first video track, decode order,
 * starting on a sync sample, as a standalone MP4 in out[0..*out_size) - sample description copied verbatim, timestamps
 * re-based to 0, coded pictures untouched.  With out == NULL only *out_size is set.  Replaces, for analysis-only runs, the
 * per-clip `ffmpeg -ss/-to ... -c:v libopenh264 -b:v 4M` re-encode of ClipTranscodingStage (clip_extraction_stages.py:318-442;
 * B200 has no NVENC, so that stage is CPU-bound there) with a memcpy of the clip's GOPs.  Host-only: ctx may be NULL. */
int cb_mp4_cut(cb_ctx* ctx, const uint8_t* data, size_t size, int first_sample, int n_samples, uint8_t* out, size_t out_cap,
               size_t* out_size);

/* 1 when the device decodes 8-bit 4:2:0 H.264 for this process (cuvidGetDecoderCaps through the libnvcuvid the decoder itself
 * loads), 0 when the driver reports no support (e.g. a container granted only the compute capability), < 0 on error
 * (libnvcuvid missing). */
int cb_nvdec_probe(cb_ctx* ctx);
/* One NVDEC session (parser + decoder + copy stream); use one per host thread, reuse it across clips. */
int cb_decoder_create(cb_ctx* ctx, cb_decoder** out);
void cb_decoder_destroy(cb_decoder* dec);
/* Decode one clip and deliver ONLY the display-order frames frame_ids[0..n_ids) (ascending; repeats allowed,
 * the counts of sample_closest) as NV12 into slots dst_slots[i] of `dst`.  Decoding stops after the last
 * wanted frame.  Replaces decode_video_cpu_frame_ids (decoder_utils.py:389-461: PyAV decodes every frame,
 * converts the wanted ones to RGB on the host) and NvVideoDecoder.generate_decoded_frames
 * (nvcodec_utils.py:247-295).  Returns only after the copies have completed. */
int cb_decoder_decode(cb_decoder* dec, const uint8_t* data, size_t size, const int32_t* frame_ids, int n_ids,
                      const cb_surface_pool* dst, const int32_t* dst_slots, cb_decode_stats* stats);

#define CB_DECODE_SEEK_SYNC 1   /* skip GOPs without a wanted frame: restart at the sync sample (stss) in front of each one */
#define CB_DECODE_DISCARD_ALL 2 /* decode every picture, deliver none (NVDEC ceiling measurement; frame_ids ignored) */
/* cb_decoder_decode with flags.  CB_DECODE_SEEK_SYNC delivers bit-identical frames while decoding only the closed GOPs
 * that contain sampled frames (streams with composition offsets fall back to sequential decode).  The reference decodes
 * every frame up to the last sampled one (decoder_utils.py:439-455); its sensor library plans sparse seeks the same way
 * (core/sensors/utils/video.py) but the clip path never got them. */
int cb_decoder_decode_ex(cb_decoder* dec, const uint8_t* data, size_t size, const int32_t* frame_ids, int n_ids,
                         const cb_surface_pool* dst, const int32_t* dst_slots, int flags, cb_decode_stats* stats);

/* Decode EVERY frame of the clip (up to max_frames) and write each as an out_w x out_h RGB u8 thumbnail into device
 * memory out[n][out_h][out_w][3]: NV12->RGB + bilinear run directly on the mapped NVDEC surface.  Replaces
 * PyNvcFrameExtractor.__call__ (nvcodec_utils.py:349-381: decode, per-frame reformat, full-resolution colour
 * convert, resize, concat) as used by VideoFrameExtractionStage for the 27x48 shot-detection frames. */
int cb_decoder_decode_thumbnails(cb_decoder* dec, const uint8_t* data, size_t size, int out_w, int out_h, uint8_t* out,
                                 int max_frames, cb_decode_stats* stats);

/* ---- shot-transition network (TransNetV2) -------------------------------------------------------- */
/* Replaces _TransNetV2.forward (cosmos_curate/models/transnetv2.py:103-148, rf=16 rl=3 rs=2 rd=1024 with frame
 * similarity + colour histograms, the only configuration the reference instantiates, :563) and the window
 * stitching of _get_predictions (pipelines/video/clipping/transnetv2_extraction_stages.py:215-264).  fp32 throughout. */
typedef struct cb_transnet cb_transnet;
int cb_transnet_create(cb_ctx* ctx, cb_transnet** out);
void cb_transnet_destroy(cb_transnet* tn);
/* Upload one tensor of the reference state_dict under its own key (host fp32, `count` elements), e.g.
 * "SDDCNN.0.DDCNN.1.Conv3D_4.layers.0.weight", "SDDCNN.2.DDCNN.0.bn.running_var", "fc1.weight",
 * "cls_layer1.bias".  cls_layer2.* and bn.num_batches_tracked are not used by forward() and are not accepted. */
int cb_transnet_set_tensor(cb_transnet* tn, const char* name, const float* data, size_t count);
/* Folds BatchNorm, repacks the convolution weights and sizes the workspace for batches of up to max_windows
 * 100-frame windows (about 150 MB per window). */
int cb_transnet_finalize(cb_transnet* tn, int max_windows);
/* The model call: windows = device uint8 [n_windows][frames_per_window][27][48][3] RGB, 1 <= frames_per_window <= 100;
 * prob_out = device fp32 [n_windows][frames_per_window], sigmoid(one_hot) of transnetv2.py:142-148. */
int cb_transnet_forward(cb_transnet* tn, const uint8_t* windows, int n_windows, int frames_per_window, float* prob_out, void* stream);
/* A whole video: frames = device uint8 [n_frames][27][48][3]; prob_out = device fp32 [n_frames], the concatenation of
 * one_hot[0, 25:75] over the reference's 100-frame / stride-50 windows (first window front-padded with frame 0,
 * the tail windows left short exactly as _get_batches leaves them).  Thresholding (prob > threshold) is the caller's. */
int cb_transnet_predict(cb_transnet* tn, const uint8_t* frames, int n_frames, float* prob_out, void* stream);

/* The network's kernels one launch at a time, each with the checks cb_transnet_forward runs before it launches them.  Every
 * pointer is device memory; a null operand or a misaligned pointer, stride or offset returns CB_ERR_ARG, zero rows is a no-op.
 *
 * The convolutions and Linear layers: out[m][out_coff + z * z_out_coff + n] = epi(sum_k A[m][k] * Wt[k][n]) for each branch z < `z`,
 * k = (tap, c) tap-major, Wt = w + z * z_w with row stride w_ld, A[m][(tap, c)] = in[src][in_coff + z * z_in_coff + c] with row stride
 * in_ld.  Row m is the position (frame m / (H W), row, col), frame t = (m / (H W)) % T of its window.
 *   mode 0: one tap, src = m.
 *   mode 1: 3 x 3 spatial taps (dh, dw) in row-major order, src = m + dh W + dw, zero outside the frame; M whole frames.
 *   mode 2: 3 temporal taps dt = (tap - 1) * (dil << (z_dil_shift ? z : 0)), src = m + dt H W, zero outside the WINDOW; M whole
 *           windows.
 * epi: fmaf(acc, scale[c], shift[c]) with scale, else acc + shift[c] (shift NULL: + 0), c = out_coff + z * z_out_coff + n; then
 * fmaxf(., 0) with relu.  in, w, out 16-byte aligned; in_ld, in_coff, out_ld, out_coff, w_ld, z_in_coff, z_out_coff and z_w multiples of
 * 4.  N must be a multiple of 4, and with cin % 16 != 0 also cin % 4 == 0 and N >= 128 (CB_ERR_UNSUPPORTED). */
typedef struct cb_transnet_conv_args {
  const float* in;
  const float* w;
  float* out;
  const float* scale; /* nullable */
  const float* shift; /* nullable */
  int M, N, cin, in_ld, in_coff, w_ld, out_ld, out_coff;
  int T, H, W, mode, dil, relu;
  int z_in_coff, z_out_coff, z_dil_shift;
  long long z_w;
} cb_transnet_conv_args;
int cb_transnet_conv(cb_ctx* ctx, const cb_transnet_conv_args* args, int z, void* stream);
/* frames uint8 [n][27][48][3]; window b < B, frame t < T is video frame first[b] + max(t - pad[b], 0) (first, pad device int32 [B]).
 * x0 fp32 [B T][27][48][4] = rgb / 255 and 0, hist fp32 [B T][512] = the L2-normalised 3-bit-per-channel RGB histogram. */
int cb_transnet_window_gather(cb_ctx* ctx, const uint8_t* frames, const int32_t* first, const int32_t* pad, int B, int T, float* x0, float* hist, void* stream);
/* out[f][ho][wo][c] (frame stride out_frame_stride floats) = 0.25 * sum over the 2 x 2 block of (relu(x2) + x1), x2 and x1 fp32
 * [frames][H][W][C]; H and W rounded down to even.  C and out_frame_stride multiples of 4. */
int cb_transnet_shortcut_pool(cb_ctx* ctx, const float* x2, const float* x1, float* out, int frames, int H, int W, int C, long long out_frame_stride, void* stream);
/* feats[f][coff + c] (row stride feats_ld) = the mean over npos >= 1 positions of x[f][p][c] (frame stride frame_stride floats). */
int cb_transnet_spatial_mean(cb_ctx* ctx, const float* x, long long frame_stride, int frames, int npos, int C, float* feats, int feats_ld, int coff, void* stream);
/* x fp32 [rows][D] in place: each row divided by max(|row|, 1e-12). */
int cb_transnet_l2_normalize_rows(cb_ctx* ctx, float* x, int rows, int D, void* stream);
/* rows = whole windows of T frames of x fp32 [rows][D]: out[r][out_coff + o] (row stride out_ld, o < 128) = relu(bias[o] + sum_j
 * sim[r][j] wt[j][o]), sim[r][j] = x[r] . x[r + j - 50] for the 101 neighbours in the same window, 0 outside it.  wt [101][128].
 * (D + 101) * 4 bytes must fit 48 KB of shared memory (CB_ERR_UNSUPPORTED). */
int cb_transnet_window_similarity_fc(cb_ctx* ctx, const float* x, int rows, int D, int T, const float* wt, const float* bias, float* out, int out_ld, int out_coff,
                                     void* stream);
/* p = sigmoid(h[r] . w + bias), h fp32 [rows][1024].  stitch 0: prob[r] = p.  stitch 1: rows are windows w0, w0 + 1, ... of T
 * frames; frames 25..74 of window w land at prob[50 w + t - 25] when that is < n_total, no other element is written. */
int cb_transnet_head(cb_ctx* ctx, const float* h, const float* w, float bias, int rows, int T, float* prob, int stitch, int w0, int n_total, void* stream);

/* ---- semantic dedup on the gathered embeddings (fp32) ------------------------------------------------ */
#define CB_ROWDOT_UPPER 1 /* a == b: only candidates i < j count (strict upper triangle) */
#define CB_ROWDOT_CLIP 2  /* clamp scores to [-1, 1] before comparing */
/* For every row j of b[nb][d]: the maximum over rows i of a[na][d] of (a_i . b_j + bias_i) and the FIRST index attaining
 * it; a candidate must be strictly greater than init_val, else out_idx[j] = -1 and out_val[j] = init_val.  All pointers
 * are device fp32 / int32, d a multiple of 16 (else CB_ERR_UNSUPPORTED); a and b must be 16-byte aligned, a null or
 * misaligned operand returns CB_ERR_ARG, nb == 0 is a no-op.  Each score is one fp32 fma chain over d in index order, then
 * + bias_i.  A candidate row holding a NaN is never returned: its NaN scores fail the `>` test; under CLIP they clamp to -1,
 * which can only be taken when init_val < -1.  Replaces the tiled `E[i0:i1] @ E[j0:j1].T -> clip -> argmax -> where`
 * loop of SemanticDedupActor.dedup (cosmos_curate/pipelines/video/dedup/dedup_actor.py:420-462) with UPPER|CLIP and
 * init_val = -1, and the nearest-centroid assignment of its KMeansMG call (:232-241) with bias_i = -|c_i|^2 / 2. */
int cb_rowdot_argmax(cb_ctx* ctx, const float* a, int na, const float* b, int nb, int d, const float* bias, int flags, float init_val, float* out_val,
                     int* out_idx, void* stream);
/* x[row] /= max(|x[row]|_2, 1e-12) in place (dedup_actor.py:224-225, :407-408); norms_out (nullable) receives |x[row]|. */
int cb_rows_l2_normalize(cb_ctx* ctx, float* x, int rows, int d, float* norms_out, void* stream);
/* sums[c][:] += sum of x[order[t]][:] for t in [seg[c], seg[c+1]): the centroid-update reduction of k-means, rows added
 * in the given order to 0.0f by one thread per (cluster, dimension), then added once to sums - bit-reproducible.  order/seg
 * are device int64.  Any n_clusters >= 1 launches (no grid limit); n_clusters or d <= 0 is CB_ERR_ARG. */
int cb_cluster_sums(cb_ctx* ctx, const float* x, const long long* order, const long long* seg, int n_clusters, int d, float* sums, void* stream);

/* ---- building blocks exported for the parity tests ------------------------------------------------ */
#define CB_EPI_NONE 0       /* C = A W^T (+ bias) */
#define CB_EPI_QUICK_GELU 1 /* C = quick_gelu(A W^T + bias) */
#define CB_EPI_GELU_TANH 2  /* C = gelu_tanh(A W^T + bias) */
#define CB_EPI_GELU_ERF 3   /* C = gelu(A W^T + bias), the exact erf form (nn.GELU()) */
/* C[M][N] = epilogue(A[M][K] . W[N][K]^T + bias[N]) (+ residual).  A, W fp16 row-major (K contiguous,
 * K % 8 == 0); bias fp32 or NULL.  If out_f32 != NULL: out_f32[M][N] (fp32) = result + (residual ?
 * residual[M][N] : 0) - residual may alias out_f32.  Else out_f16[M][N] = fp16(result).
 * The tcgen05 GEMM under every Linear of the tower (HF CLIPEncoderLayer q/k/v/out/fc1/fc2). */
int cb_gemm_f16(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* residual, float* out_f32,
                void* out_f16, int M, int N, int K, int epilogue, void* stream);
/* y[rows][d] fp16 = LayerNorm(x[rows][d] fp32) * gamma + beta. */
int cb_layernorm_f16(cb_ctx* ctx, const float* x, const float* gamma, const float* beta, void* y, int rows, int d, float eps,
                     void* stream);
/* Multi-head self-attention over qkv fp16 [n][tokens][3*hidden] (q | k | v, heads contiguous):
 * out fp16 [n][tokens][hidden]; softmax in fp32, scale = head_dim^-1/2. */
int cb_attention_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, void* stream);
/* cb_gemm_f16 plus an optional per-column fp32 scale (LayerScale, internvideo2.py:169-183): with gamma != NULL (fp32 output only),
 * out_f32 = (residual ? residual : 0) + gamma[N] * (A W^T + bias).  gamma is not folded into the fp16 weights. */
int cb_gemm_f16_ex(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* gamma, const float* residual, float* out_f32,
                   void* out_f16, int M, int N, int K, int epilogue, void* stream);
/* y[rows][d] fp16 = weight * (x * rsqrt(mean(x^2) + eps)), statistics in fp32: RMSNorm of internvideo2.py:155-166.  d % 128 == 0. */
int cb_rmsnorm_f16(cb_ctx* ctx, const float* x, const float* weight, void* y, int rows, int d, float eps, void* stream);
/* In place on qkv fp16 [rows][3*d]: the q third of each row becomes RMSNorm(q) * q_weight and the k third RMSNorm(k) * k_weight, each
 * over all d columns (every head together), fp32 statistics (Attention.qk_normalization, internvideo2.py:217-221).  d % 128 == 0. */
int cb_qk_rmsnorm_f16(cb_ctx* ctx, void* qkv, const float* q_weight, const float* k_weight, int rows, int d, float eps, void* stream);
/* Streamed attention for head_dim 88 (InternVideo2-1B: 16 heads of 88, T = 1025 at 4 frames): same layout and result as
 * cb_attention_f16 (qkv fp16 [n][tokens][3*hidden] -> out fp16 [n][tokens][hidden], scale head_dim^-1/2).  Any other head_dim:
 * CB_ERR_UNSUPPORTED.  n == 0 is a no-op. */
int cb_attention_stream_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, void* stream);
/* cb_attention_f16 for sequences padded to `tokens`: lengths is device int32 [n], and image i attends only to its keys < lengths[i]
 * (a BERT padding mask).  Keys and values past the length are never read, so whatever the padded rows hold cannot reach the output;
 * output rows past the length are zeros.  Image i's rows below its length are bitwise what the mma.sync kernel gives the unpadded
 * sequence of lengths[i] tokens, so with every length == tokens the output equals cb_attention_f16's whenever cb_attention_f16 runs
 * that kernel (outside 129..257 tokens, or always with CB_ATTN_KERNEL=mma).  Lengths outside [0, tokens] are clamped to it.
 * head_dim 64 and tokens <= 352 (K and V resident in shared memory) only; other shapes: CB_ERR_UNSUPPORTED.  n == 0 is a no-op. */
int cb_attention_masked_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, const int* lengths, void* stream);
/* Post-LN (BERT's LayerNorm(x + sublayer(x)) with the sum already in h): h[rows][d] fp32 = LayerNorm(h) * gamma + beta in place, and
 * y[rows][d] fp16 = the same values rounded.  Statistics as cb_layernorm_f16.  d % 128 == 0, d <= 1536. */
int cb_layernorm_post_f16(cb_ctx* ctx, float* h, const float* gamma, const float* beta, void* y, int rows, int d, float eps, void* stream);
/* BERT embeddings before their LayerNorm (xbert.py BertEmbeddings, token type 0): h[i][t] = (word[ids[i][t]] + type) + pos[t], fp32.
 * ids device int32 [n][L] (not range-checked here), word [vocab][d], pos [>= L][d], type [d].  d % 4 == 0. */
int cb_text_embed(cb_ctx* ctx, const int32_t* ids, const float* word, const float* pos, const float* type, float* h, int n, int L, int d,
                  void* stream);
/* The towers' row kernels, each as the tower launches it.  Every call checks its arguments before it launches: a null operand, n < 0 or a
 * misaligned pointer is CB_ERR_ARG; a width or shared-memory request the kernel cannot serve is CB_ERR_UNSUPPORTED; n == 0 is a no-op.
 * d % 128 == 0 and d <= 1536 wherever a row is a d-wide vector of float4s.
 * Tokens of the residual stream h fp32 [n][tokens][d] (tokens = grid2, or grid2 + 1 with cls fp32 [d] as token 0): h[i][t] =
 * patch[i][t'] + pos[t], then LayerNorm(.) * gamma + beta when gamma and beta are given (CLIP's pre_layrnorm; SigLIP and InternVideo2
 * pass neither).  patch fp32 [n][grid2][d], pos [tokens][d]; every pointer 16-byte aligned. */
int cb_assemble_tokens(cb_ctx* ctx, const float* patch, const float* cls, const float* pos, const float* gamma, const float* beta, float* h, int n,
                       int tokens, int grid2, int d, float eps, void* stream);
/* CLIP's pooled head on rows h + i * img_stride (img_stride >= d floats): post_layernorm, then proj fp32 [proj_dim][d] (16-byte aligned;
 * NULL: out_dim = d, no projection), emb_out [n][out_dim] = feat / |feat|, feat_out (nullable) = feat, score_out (nullable, with aes_w
 * [out_dim]) = aes_w . emb + aes_b.  (d + out_dim) * 4 bytes must fit 48 KB of shared memory. */
int cb_clip_tail(cb_ctx* ctx, const float* h, size_t img_stride, const float* gamma, const float* beta, const float* proj, int d, int proj_dim,
                 float eps, const float* aes_w, float aes_b, float* emb_out, float* feat_out, float* score_out, int n, void* stream);
/* SigLIP's MAP head attention: out fp16 [n][heads * head_dim] = softmax_t(q_h . k_t) v_t per (image, head), kv fp16 [n][tokens][2 *
 * hidden] (k | v, 4-byte aligned), q fp32 [hidden] already scaled by head_dim^-1/2.  head_dim even and <= 256. */
int cb_map_pool(cb_ctx* ctx, const void* kv, const float* q, void* out, int n, int tokens, int heads, int head_dim, void* stream);
/* emb_out [n][d] = feat / |feat| per row, feat_out (nullable) = feat, score_out (nullable, with aes_w [d]) = aes_w . emb + aes_b.
 * 1 <= d <= 1536, any width. */
int cb_l2norm_score(cb_ctx* ctx, const float* feat, int d, const float* aes_w, float aes_b, float* emb_out, float* feat_out, float* score_out, int n,
                    void* stream);
/* out fp32 [n][d] = the mean over tokens of h fp32 [n][tokens][d], tokens summed in order (tokens >= 1, n <= 65535). */
int cb_token_mean(cb_ctx* ctx, const float* h, float* out, int n, int tokens, int d, void* stream);
/* InternVideo2's attention pooling, one query per clip: out fp16 [n][hidden] = softmax_t(head_dim^-1/2 q_h . k_t) v_t per (clip, head),
 * q fp32 [n][hidden], k (4-byte aligned) and v fp16 [n][tokens][hidden].  head_dim even and <= 256. */
int cb_clip_pool(cb_ctx* ctx, const float* q, const void* k, const void* v, void* out, int n, int tokens, int heads, int head_dim, void* stream);
/* InternVideo2's patch rows: fp32 tubes [frames][3][S][S] -> fp16 [frames][(S / P)^2][k_pad], k = (c, y, x) of the P x P patch, zeros
 * from 3 P^2 to k_pad.  k_pad even and >= 3 P^2, S >= P. */
int cb_tube_patches(cb_ctx* ctx, const float* tubes, void* out, int frames, int image_size, int patch, int k_pad, void* stream);

/* ---- InternVideo2 video tower (clip embeddings) ------------------------------------------------------ */
/* The vision half of InternVideo2_Stage2.get_vid_feat (models/internvideo2_mm.py:203-217): PretrainInternVideo2.forward
 * (internvideo2.py:596-651) up to the attention-pooling clip_projector, then vision_proj and the L2 norm. */
typedef struct cb_iv2 cb_iv2;
typedef struct cb_iv2_cfg {
  int image_size, patch, frames; /* 224, 14, 4: tokens = frames * (image_size / patch)^2 + 1 */
  int hidden, layers, heads, mlp; /* 1408, 40, 16, 6144 (head_dim 88 only) */
  int clip_dim, embed_dim;        /* clip_projector output 768, vision_proj output 512 */
  float rms_eps, ln_eps;          /* 1e-6 (block and q/k RMSNorms), 1e-5 (pooling LayerNorms) */
} cb_iv2_cfg;
int cb_iv2_create(cb_ctx* ctx, const cb_iv2_cfg* cfg, cb_iv2** out);
void cb_iv2_destroy(cb_iv2* iv2);
/* Upload one named tensor (host fp32, row-major, `count` elements).  Names: patch_w[hidden][3*p*p] (Conv3d weight, k = (c, y, x)),
 * patch_b, cls, pos[tokens][hidden], L<i>.{norm1_w, qkv_w[3h][h], q_norm_w, k_norm_w, proj_w[h][h], proj_b, ls1, norm2_w,
 * fc1_w[mlp][h], fc1_b, fc2_w[h][mlp], fc2_b, ls2}, pool.{norm_q_w, norm_q_b, norm_k_w, norm_k_b, norm_v_w, norm_v_b, q_w[h][h], q_b,
 * k_w, k_b, v_w, v_b, proj_w[clip_dim][h], proj_b}, vproj_w[embed_dim][clip_dim], vproj_b.  GEMM weights are stored as fp16; norms,
 * biases, LayerScale gammas, cls and pos stay fp32.  Lifecycle: see cb_vit_set_tensor. */
int cb_iv2_set_tensor(cb_iv2* iv2, const char* name, const float* data, size_t count);
/* Checks that every tensor arrived and sizes the workspace for batches of up to max_clips clips. */
int cb_iv2_finalize(cb_iv2* iv2, int max_clips);
/* tubes: device fp32 [n][frames][3][image_size][image_size] (InternVideo2FrameCreationStage's tubes); emb_out: device fp32
 * [n][embed_dim], unit norm.  Clips are independent: an embedding does not depend on the other clips of the call. */
int cb_iv2_forward(cb_iv2* iv2, const float* tubes, int n, float* emb_out, void* stream);
/* Decoded frames to clip embeddings in one call: slots holds n_clips * frames surface indices of `pool`, clip-major (any order, repeats
 * allowed); each chunk of up to max_clips clips is one cb_video_tube_patches launch at image_size into the workspace, then the tower from
 * the patch GEMM on.  emb_out: device fp32 [n_clips][embed_dim], bitwise what cb_iv2_forward gives for cb_video_tube's tubes of the same
 * frames.  The pool's frame size is free (the frames are resized).  CB_ERR_STATE before finalize, n_clips == 0 is a no-op. */
int cb_iv2_embed_surfaces(cb_iv2* iv2, const cb_surface_pool* pool, const int32_t* slots, int n_clips, const float mean[3], const float std_[3],
                          float* emb_out, void* stream);

/* ---- InternVideo2 text tower (text embeddings) ------------------------------------------------------- */
/* InternVideo2_Stage2.get_txt_feat (models/internvideo2_mm.py:219-241) after tokenization: BertModel(mode="text") (bert/xbert.py), i.e.
 * the first `layers` (fusion_layer = 19) post-LN self-attention layers of BERT-large, the [CLS] row, text_proj and the L2 norm.  A
 * handle of its own: a caller that never embeds text never loads its weights. */
typedef struct cb_iv2_text cb_iv2_text;
typedef struct cb_iv2_text_cfg {
  int hidden, layers, heads, mlp; /* 1024, 19, 16, 4096 (head_dim 64 only) */
  int vocab, max_pos, embed_dim;  /* 30522, 512, text_proj output 512 */
  float ln_eps;                   /* 1e-12 */
} cb_iv2_text_cfg;
int cb_iv2_text_create(cb_ctx* ctx, const cb_iv2_text_cfg* cfg, cb_iv2_text** out);
void cb_iv2_text_destroy(cb_iv2_text* text);
/* Upload one named tensor (host fp32, row-major, `count` elements).  Names: tok_emb[vocab][h], pos_emb[max_pos][h], type_emb[h] (token
 * type 0), emb_ln_w, emb_ln_b, L<i>.{qkv_w[3h][h] (query | key | value), qkv_b[3h], proj_w[h][h], proj_b, ln1_w, ln1_b, fc1_w[mlp][h],
 * fc1_b, fc2_w[h][mlp], fc2_b, ln2_w, ln2_b}, tproj_w[embed_dim][h], tproj_b.  GEMM weights are stored as fp16, the rest stays fp32.
 * Lifecycle: see cb_vit_set_tensor. */
int cb_iv2_text_set_tensor(cb_iv2_text* text, const char* name, const float* data, size_t count);
/* Checks that every tensor arrived and sizes the workspace for calls of up to max_texts texts (more are run in chunks) of up to max_len
 * tokens; max_len <= min(max_pos, 352), else CB_ERR_UNSUPPORTED. */
int cb_iv2_text_finalize(cb_iv2_text* text, int max_texts, int max_len);
/* ids: HOST int32 [n][L] token ids ([CLS] ... [SEP], padded), lengths: HOST int32 [n]; emb_out: device fp32 [n][embed_dim], unit norm.
 * An id outside [0, vocab), a length outside [1, L] or L outside [1, max_pos] is CB_ERR_INVALID (nothing is launched); L > max_len is
 * CB_ERR_ARG.  A text's embedding is bitwise independent of the other texts of the call, its place among them and L. */
int cb_iv2_text_forward(cb_iv2_text* text, const int32_t* ids, const int32_t* lengths, int n, int L, float* emb_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CURATE_B200_H */
