// InternVideo2 video tower host orchestration (C ABI: cb_iv2_*): weights, workspace, layer schedule.
// Replaces InternVideo2_Stage2.get_vid_feat (cosmos_curate/models/internvideo2_mm.py:203-217) for the 1B tower
// (pretrain_internvideo2_1b_patch14_224, internvideo2.py:696-735): PretrainInternVideo2.forward up to clip_projector
// (:596-650), vision_proj, L2 norm.
//
// Per clip of T frames (tokens = T * 256 + 1, head_dim 88):
//   tube (cb_iv2_forward) or decoded surfaces (cb_iv2_embed_surfaces) -> patch rows (k = (c, y, x), padded) -> GEMM + bias -> [CLS] + pos_embed
//   40 x { RMSNorm -> qkv GEMM -> q/k RMSNorm (all heads together) -> streamed attention -> proj GEMM + bias, * ls1, + residual
//          RMSNorm -> fc1 GEMM + bias, erf GELU -> fc2 GEMM + bias, * ls2, + residual }
//   pooling: q = Wq LN_q(mean of the tokens) + bq, k = Wk LN_k(x) + bk, v = Wv LN_v(x) + bv, one query per clip, proj -> 768
//   vision_proj -> 512 -> x / |x|
// The residual stream is fp32; GEMM operands fp16 with fp32 accumulation; LayerScale in the GEMM epilogue in fp32.
#include <cuda_fp16.h>

#include "tower.h"

struct cb_iv2 {
  cb_ctx* ctx = nullptr;
  cb_iv2_cfg cfg{};
  int grid2 = 0, tokens = 0, kp = 0, k_pad = 0;
  cb::WeightStore w;
  bool finalized = false;
  int max_clips = 0;
  cb::Workspace ws;
  __half *patches = nullptr, *xn = nullptr, *qkv = nullptr, *attn = nullptr, *mlp = nullptr, *pooled_h = nullptr, *clip_h = nullptr;
  float *patch_out = nullptr, *h = nullptr, *mean = nullptr, *q = nullptr, *feat = nullptr;
};

namespace {

enum Global { PATCH_W, PATCH_B, CLS, POS, POOL_NORM_Q_W, POOL_NORM_Q_B, POOL_Q_W, POOL_Q_B, POOL_NORM_K_W, POOL_NORM_K_B, POOL_K_W, POOL_K_B,
              POOL_NORM_V_W, POOL_NORM_V_B, POOL_V_W, POOL_V_B, POOL_PROJ_W, POOL_PROJ_B, VPROJ_W, VPROJ_B, kGlobals };
enum Leaf { NORM1_W, QKV_W, Q_NORM_W, K_NORM_W, PROJ_W, PROJ_B, LS1, NORM2_W, FC1_W, FC1_B, FC2_W, FC2_B, LS2, kLeaves };

void declare_tensors(cb_iv2* v) {
  using cb::F16;
  const cb_iv2_cfg& c = v->cfg;
  const size_t d = c.hidden, m = c.mlp;
  cb::WeightStore& w = v->w;
  w.layout(kGlobals, kLeaves, c.layers);
  w.add(PATCH_W, "patch_w", d * v->kp, F16, v->kp, v->k_pad);
  w.add(PATCH_B, "patch_b", d);
  w.add(CLS, "cls", d);
  w.add(POS, "pos", (size_t)v->tokens * d);
  w.add_leaf(NORM1_W, "norm1_w", d);
  w.add_leaf(QKV_W, "qkv_w", 3 * d * d, F16);
  w.add_leaf(Q_NORM_W, "q_norm_w", d), w.add_leaf(K_NORM_W, "k_norm_w", d);
  w.add_leaf(PROJ_W, "proj_w", d * d, F16), w.add_leaf(PROJ_B, "proj_b", d);
  w.add_leaf(LS1, "ls1", d);
  w.add_leaf(NORM2_W, "norm2_w", d);
  w.add_leaf(FC1_W, "fc1_w", m * d, F16), w.add_leaf(FC1_B, "fc1_b", m);
  w.add_leaf(FC2_W, "fc2_w", d * m, F16), w.add_leaf(FC2_B, "fc2_b", d);
  w.add_leaf(LS2, "ls2", d);
  w.add(POOL_NORM_Q_W, "pool.norm_q_w", d), w.add(POOL_NORM_Q_B, "pool.norm_q_b", d), w.add(POOL_Q_W, "pool.q_w", d * d, F16), w.add(POOL_Q_B, "pool.q_b", d);
  w.add(POOL_NORM_K_W, "pool.norm_k_w", d), w.add(POOL_NORM_K_B, "pool.norm_k_b", d), w.add(POOL_K_W, "pool.k_w", d * d, F16), w.add(POOL_K_B, "pool.k_b", d);
  w.add(POOL_NORM_V_W, "pool.norm_v_w", d), w.add(POOL_NORM_V_B, "pool.norm_v_b", d), w.add(POOL_V_W, "pool.v_w", d * d, F16), w.add(POOL_V_B, "pool.v_b", d);
  w.add(POOL_PROJ_W, "pool.proj_w", (size_t)c.clip_dim * d, F16), w.add(POOL_PROJ_B, "pool.proj_b", (size_t)c.clip_dim);
  w.add(VPROJ_W, "vproj_w", (size_t)c.embed_dim * c.clip_dim, F16), w.add(VPROJ_B, "vproj_b", (size_t)c.embed_dim);
}

}  // namespace

extern "C" {

int cb_iv2_create(cb_ctx* ctx, const cb_iv2_cfg* cfg, cb_iv2** out) {
  if (!ctx) return CB_ERR_ARG;
  if (!cfg || !out) return cb::fail(ctx, CB_ERR_ARG, "iv2_create: null argument");
  *out = nullptr;
  const cb_iv2_cfg& c = *cfg;
  if (c.image_size <= 0 || c.patch <= 0 || c.image_size % c.patch || c.frames <= 0 || c.hidden <= 0 || c.layers <= 0 || c.heads <= 0 ||
      c.mlp <= 0 || c.clip_dim <= 0 || c.embed_dim <= 0 || c.hidden % c.heads)
    return cb::fail(ctx, CB_ERR_ARG, "iv2_create: inconsistent config");
  if (c.hidden / c.heads != 88) return cb::fail(ctx, CB_ERR_UNSUPPORTED, "iv2_create: head_dim %d unsupported (88 only)", c.hidden / c.heads);
  if (c.hidden % 128 || c.hidden > 1536 || c.mlp % 8 || c.clip_dim % 8 || c.embed_dim % 8)
    return cb::fail(ctx, CB_ERR_UNSUPPORTED, "iv2_create: hidden %% 128 (<= 1536), mlp, clip_dim and embed_dim %% 8 required");
  cb_iv2* v = new cb_iv2();
  v->ctx = ctx, v->cfg = c;
  const int g = c.image_size / c.patch;
  v->grid2 = c.frames * g * g;
  v->tokens = v->grid2 + 1;
  v->kp = 3 * c.patch * c.patch;
  v->k_pad = (v->kp + 63) & ~63;
  declare_tensors(v);
  *out = v;
  return CB_OK;
}

void cb_iv2_destroy(cb_iv2* v) {
  if (!v) return;
  cudaSetDevice(v->ctx->device);
  delete v;
}

int cb_iv2_set_tensor(cb_iv2* v, const char* name, const float* data, size_t count) {
  if (!v) return CB_ERR_ARG;
  v->finalized = false;
  return v->w.set(v->ctx, "iv2", name, data, count);
}

int cb_iv2_finalize(cb_iv2* v, int max_clips) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (max_clips <= 0) return cb::fail(ctx, CB_ERR_ARG, "iv2_finalize: max_clips must be positive");
  int rc;
  if ((rc = v->w.check_complete(ctx, "iv2_finalize"))) return rc;
  const cb_iv2_cfg& c = v->cfg;
  const size_t mc = max_clips, rows = mc * v->tokens, prow = mc * v->grid2, d = c.hidden;
  cb::Workspace& ws = v->ws;
  v->finalized = false;
  ws.release();
  if ((rc = ws.alloc(ctx, &v->patches, prow * v->k_pad))) return rc;
  if ((rc = ws.alloc(ctx, &v->patch_out, prow * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->h, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->xn, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->qkv, rows * 3 * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->attn, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->mlp, rows * (size_t)c.mlp))) return rc;
  if ((rc = ws.alloc(ctx, &v->mean, mc * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->q, mc * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->pooled_h, mc * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->clip_h, mc * (size_t)c.clip_dim))) return rc;
  if ((rc = ws.alloc(ctx, &v->feat, mc * (size_t)c.embed_dim))) return rc;
  v->max_clips = max_clips;
  v->finalized = true;
  return CB_OK;
}

// The tower from the n clips' patch rows in v->patches on.
static int forward_patches_chunk(cb_iv2* v, int n, float* emb, cudaStream_t s) {
  cb_ctx* ctx = v->ctx;
  const cb_iv2_cfg& c = v->cfg;
  const cb::WeightStore& w = v->w;
  const int d = c.hidden, T = v->tokens, rows = n * T, hd = d / c.heads;
  int rc;
  // patch embed: Conv3d(k = (1, p, p), stride = kernel, bias) as a GEMM over the patch rows, then [CLS] + pos_embed (no norm)
  if ((rc = cb::gemm_f16(ctx, v->patches, w.h(PATCH_W), w.f(PATCH_B), nullptr, v->patch_out, nullptr, n * v->grid2, d, v->k_pad, CB_EPI_NONE, s)))
    return rc;
  if ((rc = cb::assemble_tokens(ctx, v->patch_out, w.f(CLS), w.f(POS), nullptr, nullptr, v->h, n, T, v->grid2, d, c.ln_eps, s))) return rc;
  for (int i = 0; i < c.layers; ++i) {
    if ((rc = cb::rmsnorm_f16(ctx, v->h, w.f(i, NORM1_W), v->xn, rows, d, c.rms_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->xn, w.h(i, QKV_W), nullptr, nullptr, nullptr, v->qkv, rows, 3 * d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::qk_rmsnorm_f16(ctx, v->qkv, w.f(i, Q_NORM_W), w.f(i, K_NORM_W), rows, d, c.rms_eps, s))) return rc;
    if ((rc = cb::attention_stream_f16(ctx, v->qkv, v->attn, n, T, c.heads, hd, s))) return rc;
    if ((rc = cb::gemm_f16_ex(ctx, v->attn, w.h(i, PROJ_W), w.f(i, PROJ_B), w.f(i, LS1), v->h, v->h, nullptr, rows, d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::rmsnorm_f16(ctx, v->h, w.f(i, NORM2_W), v->xn, rows, d, c.rms_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->xn, w.h(i, FC1_W), w.f(i, FC1_B), nullptr, nullptr, v->mlp, rows, c.mlp, d, CB_EPI_GELU_ERF, s))) return rc;
    if ((rc = cb::gemm_f16_ex(ctx, v->mlp, w.h(i, FC2_W), w.f(i, FC2_B), w.f(i, LS2), v->h, v->h, nullptr, rows, d, c.mlp, CB_EPI_NONE, s)))
      return rc;
  }
  // clip_projector (AttentionPoolingBlock): the query is the token mean, keys and values get LayerNorms of their own
  __half* k = v->qkv;
  __half* val = v->qkv + (size_t)rows * d;
  if ((rc = cb::token_mean(ctx, v->h, v->mean, n, T, d, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, v->mean, w.f(POOL_NORM_Q_W), w.f(POOL_NORM_Q_B), v->pooled_h, n, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->pooled_h, w.h(POOL_Q_W), w.f(POOL_Q_B), nullptr, v->q, nullptr, n, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, v->h, w.f(POOL_NORM_K_W), w.f(POOL_NORM_K_B), v->xn, rows, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->xn, w.h(POOL_K_W), w.f(POOL_K_B), nullptr, nullptr, k, rows, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, v->h, w.f(POOL_NORM_V_W), w.f(POOL_NORM_V_B), v->xn, rows, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->xn, w.h(POOL_V_W), w.f(POOL_V_B), nullptr, nullptr, val, rows, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::clip_pool(ctx, v->q, k, val, v->pooled_h, n, T, c.heads, hd, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->pooled_h, w.h(POOL_PROJ_W), w.f(POOL_PROJ_B), nullptr, nullptr, v->clip_h, n, c.clip_dim, d, CB_EPI_NONE, s)))
    return rc;
  // vision_proj, then e / |e|
  if ((rc = cb::gemm_f16(ctx, v->clip_h, w.h(VPROJ_W), w.f(VPROJ_B), nullptr, v->feat, nullptr, n, c.embed_dim, c.clip_dim, CB_EPI_NONE, s)))
    return rc;
  return cb::l2norm_score(ctx, v->feat, c.embed_dim, nullptr, 0.f, emb, nullptr, nullptr, n, s);
}

static int forward_chunk(cb_iv2* v, const float* tubes, int n, float* emb, cudaStream_t s) {
  const int rc = cb::tube_patches(v->ctx, tubes, v->patches, n * v->cfg.frames, v->cfg.image_size, v->cfg.patch, v->k_pad, s);
  return rc ? rc : forward_patches_chunk(v, n, emb, s);
}

int cb_iv2_forward(cb_iv2* v, const float* tubes, int n, float* emb_out, void* stream) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!v->finalized) return cb::fail(ctx, CB_ERR_STATE, "iv2_forward before iv2_finalize");
  if (n < 0 || (n > 0 && (!tubes || !emb_out))) return cb::fail(ctx, CB_ERR_ARG, "iv2_forward: null argument");
  const size_t per_clip = (size_t)v->cfg.frames * 3 * v->cfg.image_size * v->cfg.image_size;
  return cb::for_chunks(n, v->max_clips, [&](int i, int m) {
    return forward_chunk(v, tubes + (size_t)i * per_clip, m, emb_out + (size_t)i * v->cfg.embed_dim, (cudaStream_t)stream);
  });
}

int cb_iv2_embed_surfaces(cb_iv2* v, const cb_surface_pool* pool, const int32_t* slots, int n_clips, const float mean[3], const float std_[3],
                          float* emb_out, void* stream) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!v->finalized) return cb::fail(ctx, CB_ERR_STATE, "iv2_embed_surfaces before iv2_finalize");
  if (n_clips < 0 || (n_clips > 0 && (!pool || !slots || !mean || !std_ || !emb_out))) return cb::fail(ctx, CB_ERR_ARG, "iv2_embed_surfaces: null argument");
  const cb_iv2_cfg& c = v->cfg;
  return cb::for_chunks(n_clips, v->max_clips, [&](int i, int m) {
    const int rc = cb::video_tube_patches(ctx, pool, slots + (size_t)i * c.frames, m * c.frames, c.image_size, c.patch, v->k_pad, mean, std_,
                                          v->patches, (cudaStream_t)stream);
    return rc ? rc : forward_patches_chunk(v, m, emb_out + (size_t)i * c.embed_dim, (cudaStream_t)stream);
  });
}

}  // extern "C"
