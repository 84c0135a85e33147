// Image tower host orchestration: weights, workspace, layer schedule (C ABI: cb_vit_*).
// Replaces transformers' CLIPModel.get_image_features as called from the reference's
// cosmos_curate/models/clip.py:71-74 and the aesthetic MLP of aesthetics.py:44-53 (folded to one affine map).
#include <cuda_fp16.h>

#include <cmath>
#include <cstring>
#include <vector>

#include "tower.h"

struct cb_vit {
  cb_ctx* ctx = nullptr;
  cb_vit_cfg cfg{};
  int grid = 0, tokens = 0, kp = 0, k_pad = 0, out_dim = 0;
  cb::WeightStore w;
  float* aes_w = nullptr;
  float aes_b = 0.f;
  bool finalized = false;
  int max_batch = 0;
  cb::Workspace ws;
  float *patch_out = nullptr, *h = nullptr;
  __half *xn = nullptr, *qkv = nullptr, *attn = nullptr, *mlp = nullptr, *patches = nullptr;
  // SigLIP MAP head: the pooling query is image-independent -> q = (probe Wq^T + bq) / sqrt(head_dim), folded at finalize
  std::vector<float> h_probe, h_wq, h_bq;
  float* map_q = nullptr;
};

namespace {

enum Global { PATCH_W, PATCH_B, POS, CLS, PRE_LN_W, PRE_LN_B, POST_LN_W, POST_LN_B, PROJ_W, MAP_PROBE, MAP_IN_W, MAP_IN_B, MAP_OUT_W,
              MAP_OUT_B, MAP_LN_W, MAP_LN_B, MAP_FC1_W, MAP_FC1_B, MAP_FC2_W, MAP_FC2_B, kGlobals };
enum Leaf { LN1_W, LN1_B, QKV_W, QKV_B, OUT_W, OUT_B, LN2_W, LN2_B, FC1_W, FC1_B, FC2_W, FC2_B, kLeaves };

void declare_tensors(cb_vit* v) {
  using cb::F16;
  const cb_vit_cfg& c = v->cfg;
  const size_t d = c.hidden, m = c.mlp;
  cb::WeightStore& w = v->w;
  w.layout(kGlobals, kLeaves, c.layers);
  w.add(PATCH_W, "patch_w", d * v->kp, F16, v->kp, v->k_pad);
  w.add(POS, "pos", (size_t)v->tokens * d);
  if (c.arch == CB_ARCH_CLIP) {
    w.add(CLS, "cls", d);
    w.add(PRE_LN_W, "pre_ln_w", d), w.add(PRE_LN_B, "pre_ln_b", d);
  } else {
    w.add(PATCH_B, "patch_b", d);
  }
  w.add_leaf(LN1_W, "ln1_w", d), w.add_leaf(LN1_B, "ln1_b", d);
  w.add_leaf(QKV_W, "qkv_w", 3 * d * d, F16), w.add_leaf(QKV_B, "qkv_b", 3 * d);
  w.add_leaf(OUT_W, "out_w", d * d, F16), w.add_leaf(OUT_B, "out_b", d);
  w.add_leaf(LN2_W, "ln2_w", d), w.add_leaf(LN2_B, "ln2_b", d);
  w.add_leaf(FC1_W, "fc1_w", m * d, F16), w.add_leaf(FC1_B, "fc1_b", m);
  w.add_leaf(FC2_W, "fc2_w", d * m, F16), w.add_leaf(FC2_B, "fc2_b", d);
  w.add(POST_LN_W, "post_ln_w", d), w.add(POST_LN_B, "post_ln_b", d);
  if (c.proj_dim > 0) w.add(PROJ_W, "proj_w", (size_t)c.proj_dim * d);
  if (c.arch == CB_ARCH_SIGLIP) {
    w.add(MAP_PROBE, "map_probe", d);
    w.add(MAP_IN_W, "map_in_w", 3 * d * d, F16), w.add(MAP_IN_B, "map_in_b", 3 * d);
    w.add(MAP_OUT_W, "map_out_w", d * d, F16), w.add(MAP_OUT_B, "map_out_b", d);
    w.add(MAP_LN_W, "map_ln_w", d), w.add(MAP_LN_B, "map_ln_b", d);
    w.add(MAP_FC1_W, "map_fc1_w", m * d, F16), w.add(MAP_FC1_B, "map_fc1_b", m);
    w.add(MAP_FC2_W, "map_fc2_w", d * m, F16), w.add(MAP_FC2_B, "map_fc2_b", d);
  }
}

}  // namespace

extern "C" {

int cb_vit_create(cb_ctx* ctx, const cb_vit_cfg* cfg, cb_vit** out) {
  if (!ctx) return CB_ERR_ARG;
  if (!cfg || !out) return cb::fail(ctx, CB_ERR_ARG, "vit_create: null argument");
  *out = nullptr;
  const cb_vit_cfg& c = *cfg;
  if (c.image_size <= 0 || c.patch <= 0 || c.image_size < c.patch || c.hidden <= 0 || c.layers <= 0 || c.heads <= 0 || c.mlp <= 0 ||
      c.hidden % c.heads)
    return cb::fail(ctx, CB_ERR_ARG, "vit_create: inconsistent config");
  if (c.arch != CB_ARCH_CLIP && c.arch != CB_ARCH_SIGLIP) return cb::fail(ctx, CB_ERR_ARG, "vit_create: unknown architecture %d", c.arch);
  if (c.arch == CB_ARCH_CLIP && c.image_size % c.patch) return cb::fail(ctx, CB_ERR_ARG, "vit_create: image_size must be a multiple of patch");
  if (c.arch == CB_ARCH_SIGLIP && c.proj_dim != 0) return cb::fail(ctx, CB_ERR_ARG, "vit_create: the SigLIP tower has no projection (proj_dim must be 0)");
  if (c.act != CB_ACT_QUICK_GELU && c.act != CB_ACT_GELU_TANH) return cb::fail(ctx, CB_ERR_ARG, "vit_create: unknown activation");
  if (c.hidden % 128 || c.mlp % 8 || (c.proj_dim % 4)) return cb::fail(ctx, CB_ERR_UNSUPPORTED, "vit_create: hidden %% 128, mlp %% 8, proj %% 4 required");
  const int hd = c.hidden / c.heads;
  if (hd % 8 || hd > 80) return cb::fail(ctx, CB_ERR_UNSUPPORTED, "vit_create: head_dim %d unsupported", hd);
  cb_vit* v = new cb_vit();
  v->ctx = ctx, v->cfg = c;
  v->grid = c.image_size / c.patch;
  v->tokens = v->grid * v->grid + (c.arch == CB_ARCH_CLIP ? 1 : 0);
  v->kp = 3 * c.patch * c.patch;
  v->k_pad = (v->kp + 63) & ~63;
  v->out_dim = c.proj_dim > 0 ? c.proj_dim : c.hidden;
  declare_tensors(v);
  *out = v;
  return CB_OK;
}

void cb_vit_destroy(cb_vit* v) {
  if (!v) return;
  cudaSetDevice(v->ctx->device);
  cudaFree(v->aes_w);
  delete v;
}

int cb_vit_k_pad(const cb_vit* v) { return v ? v->k_pad : CB_ERR_ARG; }

int cb_vit_set_tensor(cb_vit* v, const char* name, const float* data, size_t count) {
  if (!v) return CB_ERR_ARG;
  v->finalized = false;
  if (const int rc = v->w.set(v->ctx, "vit", name, data, count)) return rc;
  // host copies of the pieces the MAP query is folded from
  const size_t dd = (size_t)v->cfg.hidden;
  if (std::strcmp(name, "map_probe") == 0) v->h_probe.assign(data, data + count);
  if (std::strcmp(name, "map_in_w") == 0) v->h_wq.assign(data, data + dd * dd);
  if (std::strcmp(name, "map_in_b") == 0) v->h_bq.assign(data, data + dd);
  return CB_OK;
}

int cb_vit_set_aesthetic(cb_vit* v, const float* w, size_t count, float b) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!w || count != (size_t)v->out_dim) return cb::fail(ctx, CB_ERR_ARG, "vit_set_aesthetic: need %d weights", v->out_dim);
  if (!v->aes_w) CB_CUDA(ctx, cudaMalloc((void**)&v->aes_w, count * sizeof(float)));
  CB_CUDA(ctx, cudaMemcpy(v->aes_w, w, count * sizeof(float), cudaMemcpyHostToDevice));
  v->aes_b = b;
  return CB_OK;
}

int cb_vit_finalize(cb_vit* v, int max_batch) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (max_batch <= 0) return cb::fail(ctx, CB_ERR_ARG, "vit_finalize: max_batch must be positive");
  int rc;
  if ((rc = v->w.check_complete(ctx, "vit_finalize"))) return rc;
  const cb_vit_cfg& c = v->cfg;
  const size_t rows = (size_t)max_batch * v->tokens, prow = (size_t)max_batch * v->grid * v->grid, d = c.hidden;
  cb::Workspace& ws = v->ws;
  v->finalized = false;
  ws.release();
  if ((rc = ws.alloc(ctx, &v->patch_out, prow * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->h, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->xn, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->qkv, rows * 3 * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->attn, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->mlp, rows * (size_t)c.mlp))) return rc;
  if ((rc = ws.alloc(ctx, &v->patches, prow * (size_t)v->k_pad))) return rc;
  if (c.arch == CB_ARCH_SIGLIP) {
    const int dm = c.hidden, hd = dm / c.heads;
    std::vector<float> q(dm);
    const double sc = 1.0 / std::sqrt((double)hd);
    for (int o = 0; o < dm; ++o) {
      double acc = v->h_bq[o];
      for (int i = 0; i < dm; ++i) acc += (double)v->h_wq[(size_t)o * dm + i] * (double)v->h_probe[i];
      q[o] = (float)(acc * sc);
    }
    if ((rc = ws.alloc(ctx, &v->map_q, (size_t)dm))) return rc;
    CB_CUDA(ctx, cudaMemcpy(v->map_q, q.data(), dm * sizeof(float), cudaMemcpyHostToDevice));
  }
  v->max_batch = max_batch;
  v->finalized = true;
  return CB_OK;
}

static int forward_chunk(cb_vit* v, const void* patches, int n, float* emb, float* feat, float* score, cudaStream_t s) {
  cb_ctx* ctx = v->ctx;
  const cb_vit_cfg& c = v->cfg;
  const cb::WeightStore& w = v->w;
  const int d = c.hidden, T = v->tokens, g2 = v->grid * v->grid, rows = n * T, hd = d / c.heads;
  const int act = c.act == CB_ACT_QUICK_GELU ? CB_EPI_QUICK_GELU : CB_EPI_GELU_TANH;
  int rc;
  // patch embedding (Conv2d stride=kernel=patch as a GEMM over im2col rows), fp32 out
  if ((rc = cb::gemm_f16(ctx, patches, w.h(PATCH_W), c.arch == CB_ARCH_SIGLIP ? w.f(PATCH_B) : nullptr, nullptr, v->patch_out, nullptr, n * g2, d,
                         v->k_pad, CB_EPI_NONE, s)))
    return rc;
  if (c.arch == CB_ARCH_CLIP)
    rc = cb::assemble_tokens(ctx, v->patch_out, w.f(CLS), w.f(POS), w.f(PRE_LN_W), w.f(PRE_LN_B), v->h, n, T, g2, d, c.ln_eps, s);
  else
    rc = cb::assemble_tokens(ctx, v->patch_out, nullptr, w.f(POS), nullptr, nullptr, v->h, n, T, g2, d, c.ln_eps, s);
  if (rc) return rc;
  // CLIP reads only the [CLS] row (token 0) of the last layer's output.  Every op after that layer's attention is row-local, so
  // from there on it runs on the n [CLS] rows alone: the residual gathered into [n][d] fp32 (patch-embed output is dead by now) and
  // the attention rows into [n][d] fp16 (qkv is dead once attention has read it).
  float* h = v->h;
  __half* attn = v->attn;
  for (int i = 0; i < c.layers; ++i) {
    if ((rc = cb::layernorm_f16(ctx, v->h, w.f(i, LN1_W), w.f(i, LN1_B), v->xn, rows, d, c.ln_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->xn, w.h(i, QKV_W), w.f(i, QKV_B), nullptr, nullptr, v->qkv, rows, 3 * d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::attention_f16(ctx, v->qkv, v->attn, n, T, c.heads, hd, s))) return rc;
    int m = rows;
    if (c.arch == CB_ARCH_CLIP && i == c.layers - 1) {
      h = v->patch_out, attn = v->qkv, m = n;
      CB_CUDA(ctx, cudaMemcpy2DAsync(h, (size_t)d * sizeof(float), v->h, (size_t)T * d * sizeof(float), (size_t)d * sizeof(float), n,
                                     cudaMemcpyDeviceToDevice, s));
      CB_CUDA(ctx, cudaMemcpy2DAsync(attn, (size_t)d * sizeof(__half), v->attn, (size_t)T * d * sizeof(__half), (size_t)d * sizeof(__half), n,
                                     cudaMemcpyDeviceToDevice, s));
    }
    if ((rc = cb::gemm_f16(ctx, attn, w.h(i, OUT_W), w.f(i, OUT_B), h, h, nullptr, m, d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::layernorm_f16(ctx, h, w.f(i, LN2_W), w.f(i, LN2_B), v->xn, m, d, c.ln_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->xn, w.h(i, FC1_W), w.f(i, FC1_B), nullptr, nullptr, v->mlp, m, c.mlp, d, act, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->mlp, w.h(i, FC2_W), w.f(i, FC2_B), h, h, nullptr, m, d, c.mlp, CB_EPI_NONE, s))) return rc;
  }
  if (c.arch == CB_ARCH_CLIP)
    return cb::clip_tail(ctx, h, (size_t)d, w.f(POST_LN_W), w.f(POST_LN_B), c.proj_dim > 0 ? w.f(PROJ_W) : nullptr, d, c.proj_dim, c.ln_eps,
                         score ? v->aes_w : nullptr, v->aes_b, emb, feat, score, n, s);
  // SigLIP: post_layernorm on every token, then the MAP head (one learned query attends over the tokens, + MLP block)
  const __half* kv_w = (const __half*)w.h(MAP_IN_W) + (size_t)d * d;  // rows d..3d of in_proj_weight: K | V projections
  float* r = v->patch_out;                                             // [n][d] fp32 scratch (patch-embed output is dead by now)
  if ((rc = cb::layernorm_f16(ctx, v->h, w.f(POST_LN_W), w.f(POST_LN_B), v->xn, rows, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->xn, kv_w, w.f(MAP_IN_B) + d, nullptr, nullptr, v->qkv, rows, 2 * d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::map_pool(ctx, v->qkv, v->map_q, v->attn, n, T, c.heads, hd, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->attn, w.h(MAP_OUT_W), w.f(MAP_OUT_B), nullptr, r, nullptr, n, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, r, w.f(MAP_LN_W), w.f(MAP_LN_B), v->xn, n, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->xn, w.h(MAP_FC1_W), w.f(MAP_FC1_B), nullptr, nullptr, v->mlp, n, c.mlp, d, act, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->mlp, w.h(MAP_FC2_W), w.f(MAP_FC2_B), r, r, nullptr, n, d, c.mlp, CB_EPI_NONE, s))) return rc;
  return cb::l2norm_score(ctx, r, d, score ? v->aes_w : nullptr, v->aes_b, emb, feat, score, n, s);
}

int cb_vit_forward(cb_vit* v, const void* patches, int n, float* emb_out, float* feat_out, float* score_out, void* stream) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!v->finalized) return cb::fail(ctx, CB_ERR_STATE, "vit_forward before vit_finalize");
  if (n < 0 || (n > 0 && (!patches || !emb_out))) return cb::fail(ctx, CB_ERR_ARG, "vit_forward: null argument");
  if (score_out && !v->aes_w) return cb::fail(ctx, CB_ERR_STATE, "vit_forward: scores requested but no aesthetic head was set");
  const size_t prow = (size_t)v->grid * v->grid * v->k_pad;
  return cb::for_chunks(n, v->max_batch, [&](int i, int m) {
    return forward_chunk(v, (const __half*)patches + (size_t)i * prow, m, emb_out + (size_t)i * v->out_dim,
                         feat_out ? feat_out + (size_t)i * v->out_dim : nullptr, score_out ? score_out + i : nullptr, (cudaStream_t)stream);
  });
}

int cb_vit_embed_surfaces(cb_vit* v, const cb_surface_pool* pool, const int32_t* slots, int n, const float mean[3], const float std_[3],
                          float* emb_out, float* feat_out, float* score_out, void* stream) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!v->finalized) return cb::fail(ctx, CB_ERR_STATE, "vit_embed_surfaces before vit_finalize");
  if (n < 0 || (n > 0 && (!slots || !emb_out || !mean || !std_))) return cb::fail(ctx, CB_ERR_ARG, "vit_embed_surfaces: null argument");
  if (score_out && !v->aes_w) return cb::fail(ctx, CB_ERR_STATE, "vit_embed_surfaces: scores requested but no aesthetic head was set");
  return cb::for_chunks(n, v->max_batch, [&](int i, int m) {
    const int rc = cb::run_clip_preprocess(ctx, pool, slots + i, m, v->cfg.image_size, 2, v->cfg.patch, v->k_pad, CB_DT_F16, mean, std_, v->patches,
                                           (cudaStream_t)stream);
    return rc ? rc : forward_chunk(v, v->patches, m, emb_out + (size_t)i * v->out_dim, feat_out ? feat_out + (size_t)i * v->out_dim : nullptr,
                                   score_out ? score_out + i : nullptr, (cudaStream_t)stream);
  });
}

}  // extern "C"
