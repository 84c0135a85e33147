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

#include "tower.h"

namespace cb {
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
  cb_ctx* ctx = nullptr;
  cb_iv2_text_cfg cfg{};
  cb::WeightStore w;
  bool finalized = false;
  int max_texts = 0, max_len = 0;
  cb::Workspace ws;
  int *ids = nullptr, *lengths = nullptr;
  float *h = nullptr, *feat = nullptr;
  __half *x = nullptr, *qkv = nullptr, *attn = nullptr, *mlp = nullptr, *cls = nullptr;
};

namespace {

enum Global { TOK_EMB, POS_EMB, TYPE_EMB, EMB_LN_W, EMB_LN_B, TPROJ_W, TPROJ_B, kGlobals };
enum Leaf { QKV_W, QKV_B, PROJ_W, PROJ_B, LN1_W, LN1_B, FC1_W, FC1_B, FC2_W, FC2_B, LN2_W, LN2_B, kLeaves };

void declare_tensors(cb_iv2_text* v) {
  using cb::F16;
  const cb_iv2_text_cfg& c = v->cfg;
  const size_t d = c.hidden, m = c.mlp;
  cb::WeightStore& w = v->w;
  w.layout(kGlobals, kLeaves, c.layers);
  w.add(TOK_EMB, "tok_emb", (size_t)c.vocab * d);
  w.add(POS_EMB, "pos_emb", (size_t)c.max_pos * d);
  w.add(TYPE_EMB, "type_emb", d);  // token type 0: the only row the text path uses
  w.add(EMB_LN_W, "emb_ln_w", d), w.add(EMB_LN_B, "emb_ln_b", d);
  w.add_leaf(QKV_W, "qkv_w", 3 * d * d, F16), w.add_leaf(QKV_B, "qkv_b", 3 * d);
  w.add_leaf(PROJ_W, "proj_w", d * d, F16), w.add_leaf(PROJ_B, "proj_b", d);
  w.add_leaf(LN1_W, "ln1_w", d), w.add_leaf(LN1_B, "ln1_b", d);
  w.add_leaf(FC1_W, "fc1_w", m * d, F16), w.add_leaf(FC1_B, "fc1_b", m);
  w.add_leaf(FC2_W, "fc2_w", d * m, F16), w.add_leaf(FC2_B, "fc2_b", d);
  w.add_leaf(LN2_W, "ln2_w", d), w.add_leaf(LN2_B, "ln2_b", d);
  w.add(TPROJ_W, "tproj_w", (size_t)c.embed_dim * d, F16), w.add(TPROJ_B, "tproj_b", (size_t)c.embed_dim);
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
  declare_tensors(v);
  *out = v;
  return CB_OK;
}

void cb_iv2_text_destroy(cb_iv2_text* v) {
  if (!v) return;
  cudaSetDevice(v->ctx->device);
  delete v;
}

int cb_iv2_text_set_tensor(cb_iv2_text* v, const char* name, const float* data, size_t count) {
  if (!v) return CB_ERR_ARG;
  v->finalized = false;
  return v->w.set(v->ctx, "iv2_text", name, data, count);
}

int cb_iv2_text_finalize(cb_iv2_text* v, int max_texts, int max_len) {
  if (!v) return CB_ERR_ARG;
  cb_ctx* ctx = v->ctx;
  if (max_texts <= 0 || max_len <= 0) return cb::fail(ctx, CB_ERR_ARG, "iv2_text_finalize: max_texts and max_len must be positive");
  if (max_len > std::min(v->cfg.max_pos, kMaxResidentTokens))
    return cb::fail(ctx, CB_ERR_UNSUPPORTED, "iv2_text_finalize: max_len %d > %d", max_len, std::min(v->cfg.max_pos, kMaxResidentTokens));
  int rc;
  if ((rc = v->w.check_complete(ctx, "iv2_text_finalize"))) return rc;
  const cb_iv2_text_cfg& c = v->cfg;
  const size_t mt = max_texts, rows = mt * max_len, d = c.hidden;
  cb::Workspace& ws = v->ws;
  v->finalized = false;
  ws.release();
  if ((rc = ws.alloc(ctx, &v->ids, rows))) return rc;
  if ((rc = ws.alloc(ctx, &v->lengths, mt))) return rc;
  if ((rc = ws.alloc(ctx, &v->h, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->x, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->qkv, rows * 3 * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->attn, rows * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->mlp, rows * (size_t)c.mlp))) return rc;
  if ((rc = ws.alloc(ctx, &v->cls, mt * d))) return rc;
  if ((rc = ws.alloc(ctx, &v->feat, mt * (size_t)c.embed_dim))) return rc;
  v->max_texts = max_texts, v->max_len = max_len;
  v->finalized = true;
  return CB_OK;
}

static int text_chunk(cb_iv2_text* v, const int32_t* ids, const int32_t* lengths, int n, int L, float* emb, cudaStream_t s) {
  cb_ctx* ctx = v->ctx;
  const cb_iv2_text_cfg& c = v->cfg;
  const int d = c.hidden, rows = n * L;
  const cb::WeightStore& w = v->w;
  int rc;
  CB_CUDA(ctx, cudaMemcpyAsync(v->ids, ids, (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, s));
  CB_CUDA(ctx, cudaMemcpyAsync(v->lengths, lengths, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
  if ((rc = cb::text_embed(ctx, v->ids, w.f(TOK_EMB), w.f(POS_EMB), w.f(TYPE_EMB), v->h, n, L, d, s))) return rc;
  if ((rc = cb::layernorm_post_f16(ctx, v->h, w.f(EMB_LN_W), w.f(EMB_LN_B), v->x, rows, d, c.ln_eps, s))) return rc;
  for (int i = 0; i < c.layers; ++i) {
    if ((rc = cb::gemm_f16(ctx, v->x, w.h(i, QKV_W), w.f(i, QKV_B), nullptr, nullptr, v->qkv, rows, 3 * d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::attention_masked_f16(ctx, v->qkv, v->attn, n, L, c.heads, d / c.heads, v->lengths, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->attn, w.h(i, PROJ_W), w.f(i, PROJ_B), v->h, v->h, nullptr, rows, d, d, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::layernorm_post_f16(ctx, v->h, w.f(i, LN1_W), w.f(i, LN1_B), v->x, rows, d, c.ln_eps, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->x, w.h(i, FC1_W), w.f(i, FC1_B), nullptr, nullptr, v->mlp, rows, c.mlp, d, CB_EPI_GELU_ERF, s))) return rc;
    if ((rc = cb::gemm_f16(ctx, v->mlp, w.h(i, FC2_W), w.f(i, FC2_B), v->h, v->h, nullptr, rows, d, c.mlp, CB_EPI_NONE, s))) return rc;
    if ((rc = cb::layernorm_post_f16(ctx, v->h, w.f(i, LN2_W), w.f(i, LN2_B), v->x, rows, d, c.ln_eps, s))) return rc;
  }
  // the [CLS] row of every text -> contiguous rows, then text_proj and e / |e|
  CB_CUDA(ctx, cudaMemcpy2DAsync(v->cls, (size_t)d * sizeof(__half), v->x, (size_t)L * d * sizeof(__half), (size_t)d * sizeof(__half), n,
                                 cudaMemcpyDeviceToDevice, s));
  if ((rc = cb::gemm_f16(ctx, v->cls, w.h(TPROJ_W), w.f(TPROJ_B), nullptr, v->feat, nullptr, n, c.embed_dim, d, CB_EPI_NONE, s))) return rc;
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
  return cb::for_chunks(n, v->max_texts, [&](int i, int m) {
    return text_chunk(v, ids + (size_t)i * L, lengths + i, m, L, emb_out + (size_t)i * v->cfg.embed_dim, (cudaStream_t)stream);
  });
}

int cb_text_embed(cb_ctx* ctx, const int32_t* ids, const float* word, const float* pos, const float* type, float* h, int n, int L, int d, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::text_embed(ctx, ids, word, pos, type, h, n, L, d, (cudaStream_t)stream);
}

}  // extern "C"
