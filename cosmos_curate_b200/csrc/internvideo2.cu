// InternVideo2 video tower host orchestration (C ABI: cb_iv2_*): weights, workspace, layer schedule.
// Replaces InternVideo2_Stage2.get_vid_feat (cosmos_curate/models/internvideo2_mm.py:203-217) for the 1B tower
// (pretrain_internvideo2_1b_patch14_224, internvideo2.py:696-735): PretrainInternVideo2.forward up to clip_projector
// (:596-650), vision_proj, L2 norm.
//
// Per clip of T frames (tokens = T * 256 + 1, head_dim 88):
//   tube -> patch rows (k = (c, y, x), padded) -> GEMM + bias -> [CLS] + pos_embed
//   40 x { RMSNorm -> qkv GEMM -> q/k RMSNorm (all heads together) -> streamed attention -> proj GEMM + bias, * ls1, + residual
//          RMSNorm -> fc1 GEMM + bias, erf GELU -> fc2 GEMM + bias, * ls2, + residual }
//   pooling: q = Wq LN_q(mean of the tokens) + bq, k = Wk LN_k(x) + bk, v = Wv LN_v(x) + bv, one query per clip, proj -> 768
//   vision_proj -> 512 -> x / |x|
// The residual stream is fp32; GEMM operands fp16 with fp32 accumulation; LayerScale in the GEMM epilogue in fp32.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "common.h"

namespace cb {
int gemm_f16(cb_ctx*, const void*, const void*, const float*, const float*, float*, void*, int, int, int, int, cudaStream_t);
int gemm_f16_ex(cb_ctx*, const void*, const void*, const float*, const float*, const float*, float*, void*, int, int, int, int, cudaStream_t);
int layernorm_f16(cb_ctx*, const float*, const float*, const float*, void*, int, int, float, cudaStream_t);
int rmsnorm_f16(cb_ctx*, const float*, const float*, void*, int, int, float, cudaStream_t);
int qk_rmsnorm_f16(cb_ctx*, void*, const float*, const float*, int, int, float, cudaStream_t);
int assemble_tokens(cb_ctx*, const float*, const float*, const float*, const float*, const float*, float*, int, int, int, int, float, cudaStream_t);
int attention_stream_f16(cb_ctx*, const void*, void*, int, int, int, int, cudaStream_t);
int tube_patches(cb_ctx*, const float*, void*, int, int, int, int, cudaStream_t);
int token_mean(cb_ctx*, const float*, float*, int, int, int, cudaStream_t);
int clip_pool(cb_ctx*, const float*, const void*, const void*, void*, int, int, int, int, cudaStream_t);
int l2norm_score(cb_ctx*, const float*, int, const float*, float, float*, float*, float*, int, cudaStream_t);
}  // namespace cb

struct cb_iv2 {
  struct Tensor {
    void* d = nullptr;
    bool half = false;
  };
  cb_ctx* ctx = nullptr;
  cb_iv2_cfg cfg{};
  int grid2 = 0, tokens = 0, kp = 0, k_pad = 0;
  std::map<std::string, Tensor> t;
  bool finalized = false;
  int max_clips = 0;
  // workspace
  __half *patches = nullptr, *xn = nullptr, *qkv = nullptr, *attn = nullptr, *mlp = nullptr, *pooled_h = nullptr, *clip_h = nullptr;
  float *patch_out = nullptr, *h = nullptr, *mean = nullptr, *q = nullptr, *feat = nullptr;
  void free_workspace() {
    for (void* p : {(void*)patches, (void*)xn, (void*)qkv, (void*)attn, (void*)mlp, (void*)pooled_h, (void*)clip_h, (void*)patch_out, (void*)h,
                    (void*)mean, (void*)q, (void*)feat})
      cudaFree(p);
    patches = xn = qkv = attn = mlp = pooled_h = clip_h = nullptr;
    patch_out = h = mean = q = feat = nullptr;
  }
};

namespace {

struct Expect {
  size_t count;
  bool half;
};

std::map<std::string, Expect> expected_tensors(const cb_iv2* v) {
  const cb_iv2_cfg& c = v->cfg;
  const size_t d = c.hidden, m = c.mlp;
  std::map<std::string, Expect> e;
  e["patch_w"] = {d * (size_t)v->kp, true};
  e["patch_b"] = {d, false};
  e["cls"] = {d, false};
  e["pos"] = {(size_t)v->tokens * d, false};
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "L" + std::to_string(i) + ".";
    e[p + "norm1_w"] = {d, false};
    e[p + "qkv_w"] = {3 * d * d, true};
    e[p + "q_norm_w"] = {d, false}, e[p + "k_norm_w"] = {d, false};
    e[p + "proj_w"] = {d * d, true}, e[p + "proj_b"] = {d, false};
    e[p + "ls1"] = {d, false};
    e[p + "norm2_w"] = {d, false};
    e[p + "fc1_w"] = {m * d, true}, e[p + "fc1_b"] = {m, false};
    e[p + "fc2_w"] = {d * m, true}, e[p + "fc2_b"] = {d, false};
    e[p + "ls2"] = {d, false};
  }
  for (const char* x : {"q", "k", "v"}) {
    const std::string p = std::string("pool.");
    e[p + "norm_" + x + "_w"] = {d, false}, e[p + "norm_" + x + "_b"] = {d, false};
    e[p + x + "_w"] = {d * d, true}, e[p + x + "_b"] = {d, false};
  }
  e["pool.proj_w"] = {(size_t)c.clip_dim * d, true}, e["pool.proj_b"] = {(size_t)c.clip_dim, false};
  e["vproj_w"] = {(size_t)c.embed_dim * c.clip_dim, true}, e["vproj_b"] = {(size_t)c.embed_dim, false};
  return e;
}

template <typename T>
int dev_alloc(cb_ctx* ctx, T** p, size_t count) {
  CB_CUDA(ctx, cudaMalloc((void**)p, count * sizeof(T)));
  return CB_OK;
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
  *out = v;
  return CB_OK;
}

void cb_iv2_destroy(cb_iv2* v) {
  if (!v) return;
  cudaSetDevice(v->ctx->device);
  for (auto& kv : v->t) cudaFree(kv.second.d);
  v->free_workspace();
  delete v;
}

int cb_iv2_set_tensor(cb_iv2* v, const char* name, const float* data, size_t count) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!name || !data) return cb::fail(ctx, CB_ERR_ARG, "iv2_set_tensor: null argument");
  const auto exp = expected_tensors(v);
  const auto it = exp.find(name);
  if (it == exp.end()) return cb::fail(ctx, CB_ERR_ARG, "iv2_set_tensor: unknown tensor '%s'", name);
  if (it->second.count != count) return cb::fail(ctx, CB_ERR_ARG, "iv2_set_tensor: '%s' has %zu elements, expected %zu", name, count, it->second.count);
  cb_iv2::Tensor& t = v->t[name];
  if (t.d) cudaFree(t.d), t.d = nullptr;
  t.half = it->second.half;
  if (!t.half) {
    CB_CUDA(ctx, cudaMalloc(&t.d, count * sizeof(float)));
    CB_CUDA(ctx, cudaMemcpy(t.d, data, count * sizeof(float), cudaMemcpyHostToDevice));
    return CB_OK;
  }
  // GEMM weights: fp32 -> fp16 (round to nearest even) on the host; patch_w rows zero-padded to k_pad
  const bool is_patch = std::strcmp(name, "patch_w") == 0;
  const size_t rows = is_patch ? (size_t)v->cfg.hidden : 1, in_cols = is_patch ? (size_t)v->kp : count;
  const size_t out_cols = is_patch ? (size_t)v->k_pad : count;
  std::vector<__half> hbuf(rows * out_cols, __float2half_rn(0.f));
  for (size_t r = 0; r < rows; ++r)
    for (size_t c2 = 0; c2 < in_cols; ++c2) hbuf[r * out_cols + c2] = __float2half_rn(data[r * in_cols + c2]);
  CB_CUDA(ctx, cudaMalloc(&t.d, hbuf.size() * sizeof(__half)));
  CB_CUDA(ctx, cudaMemcpy(t.d, hbuf.data(), hbuf.size() * sizeof(__half), cudaMemcpyHostToDevice));
  return CB_OK;
}

int cb_iv2_finalize(cb_iv2* v, int max_clips) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (max_clips <= 0) return cb::fail(ctx, CB_ERR_ARG, "iv2_finalize: max_clips must be positive");
  for (auto& kv : expected_tensors(v))
    if (!v->t.count(kv.first)) return cb::fail(ctx, CB_ERR_STATE, "iv2_finalize: tensor '%s' was never set", kv.first.c_str());
  const cb_iv2_cfg& c = v->cfg;
  const size_t mc = max_clips, rows = mc * v->tokens, prow = mc * v->grid2, d = c.hidden;
  v->free_workspace();
  v->finalized = false;
  int rc;
  if ((rc = dev_alloc(ctx, &v->patches, prow * v->k_pad))) return rc;
  if ((rc = dev_alloc(ctx, &v->patch_out, prow * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->h, rows * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->xn, rows * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->qkv, rows * 3 * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->attn, rows * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->mlp, rows * (size_t)c.mlp))) return rc;
  if ((rc = dev_alloc(ctx, &v->mean, mc * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->q, mc * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->pooled_h, mc * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->clip_h, mc * (size_t)c.clip_dim))) return rc;
  if ((rc = dev_alloc(ctx, &v->feat, mc * (size_t)c.embed_dim))) return rc;
  v->max_clips = max_clips;
  v->finalized = true;
  return CB_OK;
}

static int forward_chunk(cb_iv2* v, const float* tubes, int n, float* emb, cudaStream_t s) {
  cb_ctx* ctx = v->ctx;
  const cb_iv2_cfg& c = v->cfg;
  const int d = c.hidden, T = v->tokens, rows = n * T, hd = d / c.heads;
  auto F = [&](const std::string& k) { return (const float*)v->t[k].d; };
  auto H = [&](const std::string& k) { return (const void*)v->t[k].d; };
  int rc;
  // patch embed: Conv3d(k = (1, p, p), stride = kernel, bias) as a GEMM over the patch rows, then [CLS] + pos_embed (no norm)
  if ((rc = cb::tube_patches(ctx, tubes, v->patches, n * c.frames, c.image_size, c.patch, v->k_pad, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->patches, H("patch_w"), F("patch_b"), nullptr, v->patch_out, nullptr, n * v->grid2, d, v->k_pad, CB_EPI_NONE, s)))
    return rc;
  if ((rc = cb::assemble_tokens(ctx, v->patch_out, F("cls"), F("pos"), nullptr, nullptr, v->h, n, T, v->grid2, d, c.ln_eps, s))) return rc;
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "L" + std::to_string(i) + ".";
    if ((rc = cb::rmsnorm_f16(ctx, v->h, F(p + "norm1_w"), v->xn, rows, d, c.rms_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->xn, H(p + "qkv_w"), nullptr, nullptr, nullptr, v->qkv, rows, 3 * d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::qk_rmsnorm_f16(ctx, v->qkv, F(p + "q_norm_w"), F(p + "k_norm_w"), rows, d, c.rms_eps, s))) return rc;
    if ((rc = cb::attention_stream_f16(ctx, v->qkv, v->attn, n, T, c.heads, hd, s))) return rc;
    if ((rc = cb::gemm_f16_ex(ctx, v->attn, H(p + "proj_w"), F(p + "proj_b"), F(p + "ls1"), v->h, v->h, nullptr, rows, d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::rmsnorm_f16(ctx, v->h, F(p + "norm2_w"), v->xn, rows, d, c.rms_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->xn, H(p + "fc1_w"), F(p + "fc1_b"), nullptr, nullptr, v->mlp, rows, c.mlp, d, CB_EPI_GELU_ERF, s))) return rc;
    if ((rc = cb::gemm_f16_ex(ctx, v->mlp, H(p + "fc2_w"), F(p + "fc2_b"), F(p + "ls2"), v->h, v->h, nullptr, rows, d, c.mlp, CB_EPI_NONE, s)))
      return rc;
  }
  // clip_projector (AttentionPoolingBlock): the query is the token mean, keys and values get LayerNorms of their own
  __half* k = v->qkv;
  __half* val = v->qkv + (size_t)rows * d;
  if ((rc = cb::token_mean(ctx, v->h, v->mean, n, T, d, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, v->mean, F("pool.norm_q_w"), F("pool.norm_q_b"), v->pooled_h, n, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->pooled_h, H("pool.q_w"), F("pool.q_b"), nullptr, v->q, nullptr, n, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, v->h, F("pool.norm_k_w"), F("pool.norm_k_b"), v->xn, rows, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->xn, H("pool.k_w"), F("pool.k_b"), nullptr, nullptr, k, rows, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::layernorm_f16(ctx, v->h, F("pool.norm_v_w"), F("pool.norm_v_b"), v->xn, rows, d, c.ln_eps, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->xn, H("pool.v_w"), F("pool.v_b"), nullptr, nullptr, val, rows, d, d, CB_EPI_NONE, s))) return rc;
  if ((rc = cb::clip_pool(ctx, v->q, k, val, v->pooled_h, n, T, c.heads, hd, s))) return rc;
  if ((rc = cb::gemm_f16(ctx, v->pooled_h, H("pool.proj_w"), F("pool.proj_b"), nullptr, nullptr, v->clip_h, n, c.clip_dim, d, CB_EPI_NONE, s)))
    return rc;
  // vision_proj, then e / |e|
  if ((rc = cb::gemm_f16(ctx, v->clip_h, H("vproj_w"), F("vproj_b"), nullptr, v->feat, nullptr, n, c.embed_dim, c.clip_dim, CB_EPI_NONE, s)))
    return rc;
  return cb::l2norm_score(ctx, v->feat, c.embed_dim, nullptr, 0.f, emb, nullptr, nullptr, n, s);
}

int cb_iv2_forward(cb_iv2* v, const float* tubes, int n, float* emb_out, void* stream) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!v->finalized) return cb::fail(ctx, CB_ERR_STATE, "iv2_forward before iv2_finalize");
  if (n < 0 || (n > 0 && (!tubes || !emb_out))) return cb::fail(ctx, CB_ERR_ARG, "iv2_forward: null argument");
  const size_t per_clip = (size_t)v->cfg.frames * 3 * v->cfg.image_size * v->cfg.image_size;
  for (int i = 0; i < n; i += v->max_clips) {
    const int m = std::min(v->max_clips, n - i);
    const int rc = forward_chunk(v, tubes + (size_t)i * per_clip, m, emb_out + (size_t)i * v->cfg.embed_dim, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return CB_OK;
}

}  // extern "C"
