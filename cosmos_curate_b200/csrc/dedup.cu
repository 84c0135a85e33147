// Semantic-dedup building blocks on fp32 embeddings (SURVEY.md 8f N3): the step after the embedding path.
//
// Replaces the CuPy / cuML calls of cosmos_curate/pipelines/video/dedup/dedup_actor.py:
//   :420-462  tiled  S = E[i0:i1] @ E[j0:j1].T, clip, column arg-max over earlier rows i < j, running best  (4096^2 fp32 tiles
//             materialised in HBM, ~10 elementwise passes per tile)       -> rowdot_argmax_kernel (one pass, S never leaves the SM)
//   :232-249  KMeansMG assignment (nearest centroid) and cosine distance to it -> the same kernel with a per-row bias (-|c|^2/2)
//   :224-225, :407-408  row L2 normalisation                                     -> rows_l2_normalize_kernel
//   KMeansMG centroid update                                                     -> cluster_sum_kernel (deterministic, no atomics)
// fp32 on the SIMT pipes on purpose: the pruning decision is `max cosine <= 1 - eps` on near-duplicate pairs (cosine ~ 0.99..1);
// fp16/bf16 operands (8-11 mantissa bits) would move that decision, and the reference computes it in fp32.
#include <algorithm>
#include <cmath>
#include <cstdint>

#include "common.h"

namespace cb {

struct RowdotArgs {
  const float* a;     // [na][d]  candidates (rows i)
  const float* b;     // [nb][d]  queries (columns j)
  const float* bias;  // [na] added to row i's scores, nullable
  float* out_val;     // [nb]
  int* out_idx;       // [nb]
  int na, nb, d;
  int upper;  // only candidates i < j count (strict upper triangle; a and b are the same matrix)
  int clip;   // clamp scores to [-1, 1] first (dedup_actor.py:432)
  float init_val;  // a candidate must be strictly greater than this to be taken (reference: -1.0), index -1 otherwise
};

// One CTA per 128-column tile of B; it walks the 128-row tiles of A it needs (all, or those with i < j), 128x128x16 fp32
// register-tiled products (8x8 per thread), and keeps each column's best (value, first index attaining it) in registers.
__global__ void __launch_bounds__(256) rowdot_argmax_kernel(const RowdotArgs p) {
  constexpr int BM = 128, BK = 16, LD = BM + 4;
  __shared__ __align__(16) float As[2][BK][LD];
  __shared__ __align__(16) float Bs[2][BK][LD];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int n_jt = (p.nb + BM - 1) / BM;
  const int jt = p.upper ? n_jt - 1 - (int)blockIdx.x : (int)blockIdx.x;  // triangular: heaviest column tiles first
  const int j0 = jt * BM;
  const int n_it = p.upper ? jt + 1 : (p.na + BM - 1) / BM;
  const int kchunks = p.d / BK;

  // global -> register staging: 128 rows x 16 floats = 512 float4 per operand, two per thread
  const int lrow = tid >> 2, lc4 = tid & 3;  // rows lrow and lrow + 64, float4 column lc4
  float4 ra[2], rb[2];
  auto load = [&](int i0, int kc) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + 64 * h;
      const int gi = i0 + r, gj = j0 + r;
      ra[h] = gi < p.na ? __ldg(reinterpret_cast<const float4*>(p.a + (size_t)gi * p.d + kc * BK) + lc4) : make_float4(0.f, 0.f, 0.f, 0.f);
      rb[h] = gj < p.nb ? __ldg(reinterpret_cast<const float4*>(p.b + (size_t)gj * p.d + kc * BK) + lc4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + 64 * h, c = lc4 * 4;
      As[buf][c + 0][r] = ra[h].x, As[buf][c + 1][r] = ra[h].y, As[buf][c + 2][r] = ra[h].z, As[buf][c + 3][r] = ra[h].w;
      Bs[buf][c + 0][r] = rb[h].x, Bs[buf][c + 1][r] = rb[h].y, Bs[buf][c + 2][r] = rb[h].z, Bs[buf][c + 3][r] = rb[h].w;
    }
  };

  float best_v[8];
  int best_i[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) best_v[c] = p.init_val, best_i[c] = -1;

  const int total = n_it * kchunks;
  load(0, 0);
  store(0);
  __syncthreads();
  float acc[8][8];
  for (int s = 0; s < total; ++s) {
    const int it = s / kchunks, kc = s - it * kchunks, buf = s & 1;
    if (kc == 0) {
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;
    }
    if (s + 1 < total) {
      const int it2 = (s + 1) / kchunks;
      load(it2 * BM, (s + 1) - it2 * kchunks);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]), a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]), b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w}, bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
    }
    if (kc == kchunks - 1) {  // tile finished: fold it into the running best; rows visited in ascending i, strict '>' keeps the first
      const int i0 = it * BM;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int gi = i0 + ty * 4 + (r & 3) + (r >> 2) * 64;
        if (gi >= p.na) continue;
        const float bi = p.bias ? __ldg(p.bias + gi) : 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int gj = j0 + tx * 4 + (c & 3) + (c >> 2) * 64;
          float v = acc[r][c] + bi;
          if (p.clip) v = fminf(fmaxf(v, -1.f), 1.f);
          if ((!p.upper || gi < gj) && v > best_v[c]) best_v[c] = v, best_i[c] = gi;
        }
      }
    }
    if (s + 1 < total) store(buf ^ 1);
    __syncthreads();
  }

  // the 16 threads sharing tx hold disjoint row subsets of the same 8 columns: combine (greater value, then smaller index)
  float* red_v = &As[0][0][0];                        // [16][128]
  int* red_i = reinterpret_cast<int*>(&Bs[0][0][0]);  // [16][128]
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int col = tx * 4 + (c & 3) + (c >> 2) * 64;
    red_v[ty * 128 + col] = best_v[c], red_i[ty * 128 + col] = best_i[c];
  }
  __syncthreads();
  if (tid < 128) {
    float bv = p.init_val;
    int bi = -1;
    for (int t = 0; t < 16; ++t) {
      const float v = red_v[t * 128 + tid];
      const int i = red_i[t * 128 + tid];
      if (i >= 0 && (v > bv || (v == bv && bi >= 0 && i < bi))) bv = v, bi = i;
    }
    const int gj = j0 + tid;
    if (gj < p.nb) p.out_val[gj] = bv, p.out_idx[gj] = bi;
  }
}

// x[row] /= max(||x[row]||_2, 1e-12); optionally returns the norms
__global__ void __launch_bounds__(128) rows_l2_normalize_kernel(float* __restrict__ x, int d, float* __restrict__ norms) {
  __shared__ float red[4];
  float* r = x + (size_t)blockIdx.x * d;
  float ss = 0.f;
  for (int i = threadIdx.x; i < d; i += 128) ss = fmaf(r[i], r[i], ss);
  for (int off = 16; off; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  const float nrm = sqrtf((red[0] + red[1]) + (red[2] + red[3]));
  const float denom = fmaxf(nrm, 1e-12f);
  for (int i = threadIdx.x; i < d; i += 128) r[i] = r[i] / denom;
  if (norms && threadIdx.x == 0) norms[blockIdx.x] = nrm;
}

// sums[c][:] += sum of the rows x[order[s]] for s in [seg[c], seg[c+1]) in that order (order = points sorted by label):
// one thread per (cluster, dimension), rows added sequentially -> bit-reproducible, unlike atomics.  Clusters on grid x (up to
// 2^31 - 1 of them), 256-wide dimension blocks on grid y, striding when d needs more than 65535 of them.
__global__ void __launch_bounds__(256) cluster_sum_kernel(const float* __restrict__ x, const long long* __restrict__ order, const long long* __restrict__ seg,
                                                          int d, float* __restrict__ sums) {
  const int c = blockIdx.x;
  const long long t0 = seg[c], t1 = seg[c + 1];
  for (long long dim = blockIdx.y * 256ll + threadIdx.x; dim < d; dim += gridDim.y * 256ll) {
    float s = 0.f;
    for (long long t = t0; t < t1; ++t) s += x[(size_t)order[t] * d + dim];
    sums[(size_t)c * d + dim] += s;
  }
}

}  // namespace cb

extern "C" {

int cb_rowdot_argmax(cb_ctx* ctx, const float* a, int na, const float* b, int nb, int d, const float* bias, int flags, float init_val, float* out_val,
                     int* out_idx, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  if (!a || !b || !out_val || !out_idx) return cb::fail(ctx, CB_ERR_ARG, "rowdot_argmax: null operand");
  if (((uintptr_t)a | (uintptr_t)b) & 15) return cb::fail(ctx, CB_ERR_ARG, "rowdot_argmax: a and b must be 16-byte aligned (float4 loads)");
  if (nb <= 0) return CB_OK;
  if (na < 0 || d <= 0 || d % 16) return cb::fail(ctx, CB_ERR_UNSUPPORTED, "rowdot_argmax: d=%d must be a positive multiple of 16", d);
  if ((flags & CB_ROWDOT_UPPER) && (a != b || na != nb)) return cb::fail(ctx, CB_ERR_ARG, "rowdot_argmax: CB_ROWDOT_UPPER needs a == b");
  CB_CUDA(ctx, cudaSetDevice(ctx->device));
  cb::RowdotArgs p{a, b, bias, out_val, out_idx, na, nb, d, (flags & CB_ROWDOT_UPPER) ? 1 : 0, (flags & CB_ROWDOT_CLIP) ? 1 : 0, init_val};
  cb::mark_launch(ctx, CB_PROF_CONV, (cudaStream_t)stream);
  cb::rowdot_argmax_kernel<<<(nb + 127) / 128, 256, 0, (cudaStream_t)stream>>>(p);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

int cb_rows_l2_normalize(cb_ctx* ctx, float* x, int rows, int d, float* norms_out, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  if (!x || d <= 0) return cb::fail(ctx, CB_ERR_ARG, "rows_l2_normalize: bad argument");
  if (rows <= 0) return CB_OK;
  CB_CUDA(ctx, cudaSetDevice(ctx->device));
  cb::mark_launch(ctx, CB_PROF_OTHER, (cudaStream_t)stream);
  cb::rows_l2_normalize_kernel<<<rows, 128, 0, (cudaStream_t)stream>>>(x, d, norms_out);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

int cb_cluster_sums(cb_ctx* ctx, const float* x, const long long* order, const long long* seg, int n_clusters, int d, float* sums, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  if (!x || !order || !seg || !sums || n_clusters <= 0 || d <= 0) return cb::fail(ctx, CB_ERR_ARG, "cluster_sums: bad argument");
  CB_CUDA(ctx, cudaSetDevice(ctx->device));
  cb::mark_launch(ctx, CB_PROF_OTHER, (cudaStream_t)stream);
  cb::cluster_sum_kernel<<<dim3(n_clusters, std::min((d - 1) / 256 + 1, 65535)), 256, 0, (cudaStream_t)stream>>>(x, order, seg, d, sums);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

}  // extern "C"
