// InternVideo2 text tower host orchestration (C ABI: cb_iv2_text_*): weights, workspace, layer schedule.
// Replaces InternVideo2_Stage2.get_txt_feat (cosmos_curate/models/internvideo2_mm.py:219-241): BertModel(mode="text") over the
// tokenized caption (bert/xbert.py: the first fusion_layer = 19 of BERT-large's 24 layers, self-attention only), the [CLS] row,
// text_proj, L2 norm.
//
// Per text of L tokens (ids padded to L, `length` of them real; hidden 1024 = 16 heads of 64, post-LN):
//   h = LayerNorm((word[id] + type[0]) + pos[t])                                        -> h (fp32), x (fp16 copy)
//   19 x { qkv GEMM + bias -> attention over the first `length` keys -> proj GEMM + bias + h -> LayerNorm -> h, x
//          fc1 GEMM + bias, erf GELU -> fc2 GEMM + bias + h -> LayerNorm -> h, x }
//   x[CLS] rows -> text_proj GEMM + bias -> x / |x|
// The padding mask of the reference (additive -10000 in fp32, xbert.py:1120) gives padded keys a probability of exactly 0; here
// they are never loaded.  Every row is computed on its own, so a text's embedding does not depend on L, its neighbours or its slot.
#include <cuda_fp16.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "common.h"

namespace cb {
int gemm_f16(cb_ctx*, const void*, const void*, const float*, const float*, float*, void*, int, int, int, int, cudaStream_t);
int layernorm_post_f16(cb_ctx*, float*, const float*, const float*, void*, int, int, float, cudaStream_t);
int attention_masked_f16(cb_ctx*, const void*, void*, int, int, int, int, const int*, cudaStream_t);
int l2norm_score(cb_ctx*, const float*, int, const float*, float, float*, float*, float*, int, cudaStream_t);

// h[n * L + t] = (word[ids[n * L + t]] + type) + pos[t], fp32; one warp per row.  Ids are checked on the host.
__global__ void __launch_bounds__(256) text_embed_kernel(const int* __restrict__ ids, const float* __restrict__ word, const float* __restrict__ pos,
                                                         const float* __restrict__ type, float* __restrict__ h, int rows, int L, int d) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int t = row % L;
  const float4* w = (const float4*)(word + (size_t)ids[row] * d);
  const float4* p = (const float4*)(pos + (size_t)t * d);
  const float4* ty = (const float4*)type;
  float4* out = (float4*)(h + (size_t)row * d);
  for (int i = lane; i < (d >> 2); i += 32) {
    const float4 a = __ldg(w + i), b = __ldg(ty + i), c = __ldg(p + i);
    out[i] = make_float4((a.x + b.x) + c.x, (a.y + b.y) + c.y, (a.z + b.z) + c.z, (a.w + b.w) + c.w);
  }
}

int text_embed(cb_ctx* ctx, const int* ids, const float* word, const float* pos, const float* type, float* h, int n, int L, int d, cudaStream_t stream) {
  if (!ids || !word || !pos || !type || !h) return fail(ctx, CB_ERR_ARG, "text_embed: null operand");
  if (n < 0 || L <= 0 || d <= 0 || d % 4) return fail(ctx, CB_ERR_ARG, "text_embed: n=%d L=%d d=%d", n, L, d);
  const int rows = n * L;
  if (rows == 0) return CB_OK;
  mark_launch(ctx, CB_PROF_OTHER, stream);
  text_embed_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(ids, word, pos, type, h, rows, L, d);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}
}  // namespace cb

struct cb_iv2_text {
  struct Tensor {
    void* d = nullptr;
    bool half = false;
  };
  cb_ctx* ctx = nullptr;
  cb_iv2_text_cfg cfg{};
  std::map<std::string, Tensor> t;
  bool finalized = false;
  int max_texts = 0, max_len = 0;
  // workspace
  int *ids = nullptr, *lengths = nullptr;
  float *h = nullptr, *feat = nullptr;
  __half *x = nullptr, *qkv = nullptr, *attn = nullptr, *mlp = nullptr, *cls = nullptr;
  void free_workspace() {
    for (void* p : {(void*)ids, (void*)lengths, (void*)h, (void*)feat, (void*)x, (void*)qkv, (void*)attn, (void*)mlp, (void*)cls}) cudaFree(p);
    ids = lengths = nullptr;
    h = feat = nullptr;
    x = qkv = attn = mlp = cls = nullptr;
  }
};

namespace {

struct Expect {
  size_t count;
  bool half;
};

std::map<std::string, Expect> expected_tensors(const cb_iv2_text* v) {
  const cb_iv2_text_cfg& c = v->cfg;
  const size_t d = c.hidden, m = c.mlp;
  std::map<std::string, Expect> e;
  e["tok_emb"] = {(size_t)c.vocab * d, false};
  e["pos_emb"] = {(size_t)c.max_pos * d, false};
  e["type_emb"] = {d, false};  // token type 0: the only row the text path uses
  e["emb_ln_w"] = {d, false}, e["emb_ln_b"] = {d, false};
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "L" + std::to_string(i) + ".";
    e[p + "qkv_w"] = {3 * d * d, true}, e[p + "qkv_b"] = {3 * d, false};
    e[p + "proj_w"] = {d * d, true}, e[p + "proj_b"] = {d, false};
    e[p + "ln1_w"] = {d, false}, e[p + "ln1_b"] = {d, false};
    e[p + "fc1_w"] = {m * d, true}, e[p + "fc1_b"] = {m, false};
    e[p + "fc2_w"] = {d * m, true}, e[p + "fc2_b"] = {d, false};
    e[p + "ln2_w"] = {d, false}, e[p + "ln2_b"] = {d, false};
  }
  e["tproj_w"] = {(size_t)c.embed_dim * d, true}, e["tproj_b"] = {(size_t)c.embed_dim, false};
  return e;
}

template <typename T>
int dev_alloc(cb_ctx* ctx, T** p, size_t count) {
  CB_CUDA(ctx, cudaMalloc((void**)p, count * sizeof(T)));
  return CB_OK;
}

constexpr int kMaxResidentTokens = 352;  // attention_masked_f16 keeps every key of a sequence in shared memory

}  // namespace

extern "C" {

int cb_iv2_text_create(cb_ctx* ctx, const cb_iv2_text_cfg* cfg, cb_iv2_text** out) {
  if (!ctx) return CB_ERR_ARG;
  if (!cfg || !out) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_create: null argument");
  *out = nullptr;
  const cb_iv2_text_cfg& c = *cfg;
  if (c.hidden <= 0 || c.layers <= 0 || c.heads <= 0 || c.mlp <= 0 || c.vocab <= 0 || c.max_pos <= 0 || c.embed_dim <= 0 || c.hidden % c.heads)
    return cb::fail(ctx, CB_ERR_ARG, "iv2_text_create: inconsistent config");
  if (c.hidden / c.heads != 64) return cb::fail(ctx, CB_ERR_UNSUPPORTED, "iv2_text_create: head_dim %d unsupported (64 only)", c.hidden / c.heads);
  if (c.hidden % 128 || c.hidden > 1536 || c.mlp % 8 || c.embed_dim % 8)
    return cb::fail(ctx, CB_ERR_UNSUPPORTED, "iv2_text_create: hidden %% 128 (<= 1536), mlp and embed_dim %% 8 required");
  cb_iv2_text* v = new cb_iv2_text();
  v->ctx = ctx, v->cfg = c;
  *out = v;
  return CB_OK;
}

void cb_iv2_text_destroy(cb_iv2_text* v) {
  if (!v) return;
  cudaSetDevice(v->ctx->device);
  for (auto& kv : v->t) cudaFree(kv.second.d);
  v->free_workspace();
  delete v;
}

int cb_iv2_text_set_tensor(cb_iv2_text* v, const char* name, const float* data, size_t count) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!name || !data) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_set_tensor: null argument");
  const auto exp = expected_tensors(v);
  const auto it = exp.find(name);
  if (it == exp.end()) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_set_tensor: unknown tensor '%s'", name);
  if (it->second.count != count)
    return cb::fail(ctx, CB_ERR_ARG, "iv2_text_set_tensor: '%s' has %zu elements, expected %zu", name, count, it->second.count);
  cb_iv2_text::Tensor& t = v->t[name];
  if (t.d) cudaFree(t.d), t.d = nullptr;
  t.half = it->second.half;
  if (!t.half) {
    CB_CUDA(ctx, cudaMalloc(&t.d, count * sizeof(float)));
    CB_CUDA(ctx, cudaMemcpy(t.d, data, count * sizeof(float), cudaMemcpyHostToDevice));
    return CB_OK;
  }
  std::vector<__half> hbuf(count);  // GEMM weights: fp32 -> fp16, round to nearest even
  for (size_t i = 0; i < count; ++i) hbuf[i] = __float2half_rn(data[i]);
  CB_CUDA(ctx, cudaMalloc(&t.d, count * sizeof(__half)));
  CB_CUDA(ctx, cudaMemcpy(t.d, hbuf.data(), count * sizeof(__half), cudaMemcpyHostToDevice));
  return CB_OK;
}

int cb_iv2_text_finalize(cb_iv2_text* v, int max_texts, int max_len) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (max_texts <= 0 || max_len <= 0) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_finalize: max_texts and max_len must be positive");
  if (max_len > std::min(v->cfg.max_pos, kMaxResidentTokens))
    return cb::fail(ctx, CB_ERR_UNSUPPORTED, "iv2_text_finalize: max_len %d > %d", max_len, std::min(v->cfg.max_pos, kMaxResidentTokens));
  for (auto& kv : expected_tensors(v))
    if (!v->t.count(kv.first)) return cb::fail(ctx, CB_ERR_STATE, "iv2_text_finalize: tensor '%s' was never set", kv.first.c_str());
  const cb_iv2_text_cfg& c = v->cfg;
  const size_t mt = max_texts, rows = mt * max_len, d = c.hidden;
  v->free_workspace();
  v->finalized = false;
  int rc;
  if ((rc = dev_alloc(ctx, &v->ids, rows))) return rc;
  if ((rc = dev_alloc(ctx, &v->lengths, mt))) return rc;
  if ((rc = dev_alloc(ctx, &v->h, rows * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->x, rows * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->qkv, rows * 3 * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->attn, rows * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->mlp, rows * (size_t)c.mlp))) return rc;
  if ((rc = dev_alloc(ctx, &v->cls, mt * d))) return rc;
  if ((rc = dev_alloc(ctx, &v->feat, mt * (size_t)c.embed_dim))) return rc;
  v->max_texts = max_texts, v->max_len = max_len;
  v->finalized = true;
  return CB_OK;
}

static int text_chunk(cb_iv2_text* v, const int32_t* ids, const int32_t* lengths, int n, int L, float* emb, cudaStream_t s) {
  cb_ctx* ctx = v->ctx;
  const cb_iv2_text_cfg& c = v->cfg;
  const int d = c.hidden, rows = n * L;
  auto F = [&](const std::string& k) { return (const float*)v->t[k].d; };
  auto H = [&](const std::string& k) { return (const void*)v->t[k].d; };
  int rc;
  CB_CUDA(ctx, cudaMemcpyAsync(v->ids, ids, (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, s));
  CB_CUDA(ctx, cudaMemcpyAsync(v->lengths, lengths, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
  if ((rc = cb::text_embed(ctx, v->ids, F("tok_emb"), F("pos_emb"), F("type_emb"), v->h, n, L, d, s))) return rc;
  if ((rc = cb::layernorm_post_f16(ctx, v->h, F("emb_ln_w"), F("emb_ln_b"), v->x, rows, d, c.ln_eps, s))) return rc;
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "L" + std::to_string(i) + ".";
    if ((rc = cb::gemm_f16(ctx, v->x, H(p + "qkv_w"), F(p + "qkv_b"), nullptr, nullptr, v->qkv, rows, 3 * d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::attention_masked_f16(ctx, v->qkv, v->attn, n, L, c.heads, d / c.heads, v->lengths, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->attn, H(p + "proj_w"), F(p + "proj_b"), v->h, v->h, nullptr, rows, d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::layernorm_post_f16(ctx, v->h, F(p + "ln1_w"), F(p + "ln1_b"), v->x, rows, d, c.ln_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->x, H(p + "fc1_w"), F(p + "fc1_b"), nullptr, nullptr, v->mlp, rows, c.mlp, d, CB_EPI_GELU_ERF, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->mlp, H(p + "fc2_w"), F(p + "fc2_b"), v->h, v->h, nullptr, rows, d, c.mlp, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::layernorm_post_f16(ctx, v->h, F(p + "ln2_w"), F(p + "ln2_b"), v->x, rows, d, c.ln_eps, s))) return rc;
  }
  // the [CLS] row of every text -> contiguous rows, then text_proj and e / |e|
  CB_CUDA(ctx, cudaMemcpy2DAsync(v->cls, (size_t)d * sizeof(__half), v->x, (size_t)L * d * sizeof(__half), (size_t)d * sizeof(__half), n,
                                 cudaMemcpyDeviceToDevice, s));
  if ((rc = cb::gemm_f16(ctx, v->cls, H("tproj_w"), F("tproj_b"), nullptr, v->feat, nullptr, n, c.embed_dim, d, CB_EPI_NONE, s))) return rc;
  return cb::l2norm_score(ctx, v->feat, c.embed_dim, nullptr, 0.f, emb, nullptr, nullptr, n, s);
}

int cb_iv2_text_forward(cb_iv2_text* v, const int32_t* ids, const int32_t* lengths, int n, int L, float* emb_out, void* stream) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (!v->finalized) return cb::fail(ctx, CB_ERR_STATE, "iv2_text_forward before iv2_text_finalize");
  if (n < 0 || (n > 0 && (!ids || !lengths || !emb_out))) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_forward: null argument");
  if (n == 0) return CB_OK;
  if (L < 1 || L > v->cfg.max_pos) return cb::fail(ctx, CB_ERR_INVALID, "iv2_text_forward: L=%d outside [1, %d]", L, v->cfg.max_pos);
  if (L > v->max_len) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_forward: L=%d exceeds the workspace's max_len %d", L, v->max_len);
  for (int i = 0; i < n; ++i) {
    if (lengths[i] < 1 || lengths[i] > L) return cb::fail(ctx, CB_ERR_INVALID, "iv2_text_forward: text %d has length %d outside [1, %d]", i, lengths[i], L);
    for (int j = 0; j < L; ++j) {
      const int32_t id = ids[(size_t)i * L + j];
      if (id < 0 || id >= v->cfg.vocab) return cb::fail(ctx, CB_ERR_INVALID, "iv2_text_forward: text %d token %d has id %d outside [0, %d)", i, j, id, v->cfg.vocab);
    }
  }
  for (int i = 0; i < n; i += v->max_texts) {
    const int m = std::min(v->max_texts, n - i);
    const int rc = text_chunk(v, ids + (size_t)i * L, lengths + i, m, L, emb_out + (size_t)i * v->cfg.embed_dim, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return CB_OK;
}

int cb_text_embed(cb_ctx* ctx, const int32_t* ids, const float* word, const float* pos, const float* type, float* h, int n, int L, int d, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::text_embed(ctx, ids, word, pos, type, h, n, L, d, (cudaStream_t)stream);
}

}  // extern "C"
