// TransNetV2 shot-transition network in fp32 on the SIMT pipes (SURVEY.md 8a row a10, 8f N1).
//
// Replaces  _TransNetV2.forward (cosmos_curate/models/transnetv2.py:103-148) and the windowing of _get_predictions
// (pipelines/video/clipping/transnetv2_extraction_stages.py:215-264).  The shot boundaries derived from the output must
// be the reference's, so the whole net stays in fp32 with fp32 accumulation (no fp16/tf32 tensor-core path: a 1e-3
// error on a probability next to the 0.4 threshold moves a boundary).
//
// Activations are frame-major, channels-last: [window][frame][row][col][channel] fp32, i.e. a matrix
// [M = B*T*H*W positions][C].  Every convolution is a gather-GEMM over that matrix:
//   (1,3,3) conv of the four dilation branches at once : A = 9 spatial taps x Cin  (zero outside the frame),  N = 4 * 2F
//   (3,1,1) conv, one branch per blockIdx.z            : A = 3 temporal taps x 2F (zero outside the WINDOW),  N = F
//   Linear layers (similarity projection, fc1)         : A = the rows themselves
// BatchNorm3d (eval, eps 1e-3) is folded into a per-channel scale/shift applied in the epilogue of the temporal conv.
#include <cmath>
#include <cstring>
#include <string>

#include "common.h"

namespace cb {

constexpr int kFrameH = 27, kFrameW = 48, kLookup = 101, kStacks = 3, kBlocks = 2, kBranches = 4;
constexpr int kSimDim = 128, kHistBins = 512, kFcIn = 4864, kFcOut = 1024, kTrunkOff = 256;

struct ConvGemmArgs {
  const float* in;
  const float* w;
  float* out;
  const float* scale;  // nullable, indexed by output channel (out_coff + n)
  const float* shift;  // nullable
  int M, N, cin, in_ld, in_coff, w_ld, out_ld, out_coff;
  int T, H, W;  // frames per window, frame size (a row of the matrix is one (frame,row,col) position)
  int mode;     // 0 rows as they are, 1 = 3x3 spatial taps, 2 = 3 temporal taps with dilation `dil`
  int dil, relu;
  int z_in_coff, z_out_coff;  // per-blockIdx.z increments (the four dilation branches in one launch)
  int z_dil_shift;            // dilation = dil << blockIdx.z
  long long z_w;
};

// C[M,N] = gather(A)[M, taps*cin] * Wt[taps*cin, N].  256 threads as (256/CT) x CT; each thread owns an 8 x TN block, so the
// CTA tile is BM = 8*256/CT rows by BN = CT*TN columns: 128x128 for the wide spatial convs, 512x16 / 256x32 / 256x64 for the
// narrow temporal ones (a 128x16 tile would spend its time on shared-memory loads: 8 FMAs per 3 loads).  K is walked in
// chunks of BKC channels of one tap.  Register-staged double buffering: the next chunk's global loads are in flight during
// the FMAs.  The k order of every output's sum does not depend on the tile shape, so all variants give identical bits.
template <int CT, int TN, int BKC>
__global__ void __launch_bounds__(256) conv_gemm_kernel(const ConvGemmArgs a) {
  constexpr int TM = 8, RT = 256 / CT, BM = RT * TM, BN = CT * TN, LDA = BM + 4, HALF_M = BM / 2, HALF_N = BN / 2;
  constexpr int A_F4 = BM * BKC / 4, A_IT = (A_F4 + 255) / 256, B_F4 = BKC * BN / 4, B_IT = (B_F4 + 255) / 256;
  constexpr int KC4 = BKC / 4, BN4 = BN / 4;
  static_assert(TN == 4 || TN == 8, "TN");
  __shared__ __align__(16) float As[2][BKC][LDA];
  __shared__ __align__(16) float Bs[2][BKC][BN];
  const int tid = threadIdx.x, ty = tid / CT, tx = tid % CT;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN, z = blockIdx.z;
  const float* __restrict__ in = a.in + a.in_coff + z * a.z_in_coff;
  const float* __restrict__ wt = a.w + (long long)z * a.z_w;
  const int HW = a.H * a.W;
  const int dil = a.dil << (a.z_dil_shift ? z : 0);

  int a_m[A_IT], a_t[A_IT], a_h[A_IT], a_w[A_IT], a_row[A_IT], a_c4[A_IT];
  bool a_ok[A_IT];
#pragma unroll
  for (int it = 0; it < A_IT; ++it) {
    const int idx = tid + it * 256;
    a_row[it] = idx / KC4, a_c4[it] = idx % KC4;
    const int m = m0 + a_row[it];
    a_ok[it] = idx < A_F4 && m < a.M;
    const int f = m / HW, hw = m - f * HW;
    a_m[it] = m, a_t[it] = f % a.T, a_h[it] = hw / a.W, a_w[it] = hw - (hw / a.W) * a.W;
  }
  const int taps = a.mode == 1 ? 9 : (a.mode == 2 ? 3 : 1);
  const int chunks_per_tap = a.cin / BKC, n_chunks = taps * chunks_per_tap;

  float4 ra[A_IT], rb[B_IT];
  auto load_chunk = [&](int kc) {
    const int tap = kc / chunks_per_tap, c0 = (kc - tap * chunks_per_tap) * BKC;
#pragma unroll
    for (int it = 0; it < A_IT; ++it) {
      bool ok = a_ok[it];
      long long src = a_m[it];
      if (a.mode == 1) {
        const int dh = tap / 3 - 1, dw = tap % 3 - 1;
        ok = ok && (unsigned)(a_h[it] + dh) < (unsigned)a.H && (unsigned)(a_w[it] + dw) < (unsigned)a.W;
        src += dh * a.W + dw;
      } else if (a.mode == 2) {
        const int dt = (tap - 1) * dil;
        ok = ok && (unsigned)(a_t[it] + dt) < (unsigned)a.T;
        src += (long long)dt * HW;
      }
      ra[it] = ok ? __ldg(reinterpret_cast<const float4*>(in + src * a.in_ld + c0 + a_c4[it] * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int it = 0; it < B_IT; ++it) {
      const int idx = tid + it * 256, k = idx / BN4, n4 = idx % BN4;
      const bool ok = idx < B_F4 && n0 + n4 * 4 < a.N;
      rb[it] = ok ? __ldg(reinterpret_cast<const float4*>(wt + (long long)(kc * BKC + k) * a.w_ld + n0 + n4 * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_chunk = [&](int buf) {
#pragma unroll
    for (int it = 0; it < A_IT; ++it) {
      if (tid + it * 256 < A_F4) {
        const int r = a_row[it], c = a_c4[it] * 4;
        As[buf][c + 0][r] = ra[it].x, As[buf][c + 1][r] = ra[it].y, As[buf][c + 2][r] = ra[it].z, As[buf][c + 3][r] = ra[it].w;
      }
    }
#pragma unroll
    for (int it = 0; it < B_IT; ++it) {
      const int idx = tid + it * 256;
      if (idx < B_F4) *reinterpret_cast<float4*>(&Bs[buf][idx / BN4][(idx % BN4) * 4]) = rb[it];
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_chunk(0);
  store_chunk(0);
  __syncthreads();
  for (int kc = 0; kc < n_chunks; ++kc) {
    const int buf = kc & 1;
    if (kc + 1 < n_chunks) load_chunk(kc + 1);
#pragma unroll
    for (int k = 0; k < BKC; ++k) {
      float av[TM], bv[TN];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][HALF_M + ty * 4]);
      av[0] = a0.x, av[1] = a0.y, av[2] = a0.z, av[3] = a0.w, av[4] = a1.x, av[5] = a1.y, av[6] = a1.z, av[7] = a1.w;
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      bv[0] = b0.x, bv[1] = b0.y, bv[2] = b0.z, bv[3] = b0.w;
      if constexpr (TN == 8) {
        const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][HALF_N + tx * 4]);
        bv[4] = b1.x, bv[5] = b1.y, bv[6] = b1.z, bv[7] = b1.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kc + 1 < n_chunks) store_chunk(buf ^ 1);
    __syncthreads();
  }

  // epilogue: BatchNorm scale/shift or bias, optional ReLU
  const int ocoff = a.out_coff + z * a.z_out_coff;
  float sc[TN], sh[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) {
    const int n = n0 + tx * 4 + (j & 3) + (j >> 2) * HALF_N;
    const bool ok = n < a.N;
    sc[j] = (ok && a.scale) ? __ldg(a.scale + ocoff + n) : 1.f;
    sh[j] = (ok && a.shift) ? __ldg(a.shift + ocoff + n) : 0.f;
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * 4 + (i & 3) + (i >> 2) * HALF_M;
    if (m >= a.M) continue;
    float* orow = a.out + (long long)m * a.out_ld + ocoff + n0;
    float v[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      float y = a.scale ? fmaf(acc[i][j], sc[j], sh[j]) : acc[i][j] + sh[j];
      v[j] = a.relu ? fmaxf(y, 0.f) : y;
    }
    if (n0 + tx * 4 < a.N) *reinterpret_cast<float4*>(orow + tx * 4) = make_float4(v[0], v[1], v[2], v[3]);
    if constexpr (TN == 8) {
      if (n0 + HALF_N + tx * 4 < a.N) *reinterpret_cast<float4*>(orow + HALF_N + tx * 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
}

// uint8 frames of one video -> fp32/255 window tensor [B][T][27][48][4] (4th channel zero), and the per-frame 512-bin
// colour histogram, L2-normalised (transnetv2.py:108-113, :440-486).  Window b holds video frames
// first[b] + max(t - pad[b], 0): front padding repeats the first frame (transnetv2_extraction_stages.py:226-231).
__global__ void __launch_bounds__(256) window_gather_kernel(const uint8_t* __restrict__ frames, const int* __restrict__ first, const int* __restrict__ pad,
                                                            int T, float* __restrict__ x0, float* __restrict__ hist) {
  constexpr int NPIX = kFrameH * kFrameW;
  __shared__ int bins[kHistBins];
  __shared__ float red[8];
  const int b = blockIdx.x / T, t = blockIdx.x % T, tid = threadIdx.x;
  const int src = first[b] + max(t - pad[b], 0);
  const uint8_t* f = frames + (size_t)src * NPIX * 3;
  for (int i = tid; i < kHistBins; i += 256) bins[i] = 0;
  __syncthreads();
  float4* o = reinterpret_cast<float4*>(x0) + (size_t)blockIdx.x * NPIX;
  for (int p = tid; p < NPIX; p += 256) {
    const int r = f[p * 3], g = f[p * 3 + 1], bl = f[p * 3 + 2];
    o[p] = make_float4((float)r / 255.0f, (float)g / 255.0f, (float)bl / 255.0f, 0.f);
    atomicAdd(&bins[((r >> 5) << 6) + ((g >> 5) << 3) + (bl >> 5)], 1);
  }
  __syncthreads();
  // sum of squares of integer counts <= 1296^2 < 2^24: exact in fp32 in any order
  float ss = 0.f;
  for (int i = tid; i < kHistBins; i += 256) ss += (float)bins[i] * (float)bins[i];
  for (int off = 16; off; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float denom = fmaxf(sqrtf(tot), 1e-12f);
  for (int i = tid; i < kHistBins; i += 256) hist[(size_t)blockIdx.x * kHistBins + i] = (float)bins[i] / denom;
}

// StackedDDCNNV2 tail (transnetv2.py:204-221): y = relu(block2) + block1, then 2x2 spatial average pooling (floor).
__global__ void __launch_bounds__(256) shortcut_pool_kernel(const float* __restrict__ x2, const float* __restrict__ x1, float* __restrict__ out, int frames, int H,
                                                            int W, int C, long long out_frame_stride) {
  const int Hp = H / 2, Wp = W / 2, C4 = C / 4;
  const long long total = (long long)frames * Hp * Wp * C4;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c4 = (int)(i % C4);
    long long r = i / C4;
    const int wo = (int)(r % Wp);
    r /= Wp;
    const int ho = (int)(r % Hp), f = (int)(r / Hp);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const long long p = (((long long)f * H + 2 * ho + dy) * W + 2 * wo + dx) * C4 + c4;
        const float4 a = __ldg(reinterpret_cast<const float4*>(x2) + p), b = __ldg(reinterpret_cast<const float4*>(x1) + p);
        s.x += fmaxf(a.x, 0.f) + b.x, s.y += fmaxf(a.y, 0.f) + b.y, s.z += fmaxf(a.z, 0.f) + b.z, s.w += fmaxf(a.w, 0.f) + b.w;
      }
    float4* o = reinterpret_cast<float4*>(out + (long long)f * out_frame_stride + ((long long)ho * Wp + wo) * C) + c4;
    *o = make_float4(s.x * 0.25f, s.y * 0.25f, s.z * 0.25f, s.w * 0.25f);
  }
}

// mean over the pooled frame of every channel -> feats[frame][coff + c] (FrameSimilarity input, transnetv2.py:387)
__global__ void __launch_bounds__(128) spatial_mean_kernel(const float* __restrict__ x, long long frame_stride, int npos, int C, float* __restrict__ feats,
                                                           int feats_ld, int coff) {
  const int f = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += 128) {
    float s = 0.f;
    for (int p = 0; p < npos; ++p) s += x[(long long)f * frame_stride + (long long)p * C + c];
    feats[(long long)f * feats_ld + coff + c] = s / (float)npos;
  }
}

// rows /= max(||row||_2, 1e-12)  (functional.normalize, transnetv2.py:391)
__global__ void __launch_bounds__(128) l2_normalize_rows_kernel(float* __restrict__ x, int D) {
  __shared__ float red[4];
  float* r = x + (long long)blockIdx.x * D;
  float ss = 0.f;
  for (int i = threadIdx.x; i < D; i += 128) ss += r[i] * r[i];
  for (int off = 16; off; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  const float denom = fmaxf(sqrtf(red[0] + red[1] + red[2] + red[3]), 1e-12f);
  for (int i = threadIdx.x; i < D; i += 128) r[i] = r[i] / denom;
}

// One block per (window, frame): cosine similarities to the 101 neighbours t-50..t+50 inside the window (zero outside),
// then Linear(101 -> 128) + ReLU into the concat row (transnetv2.py:393-418 and :503-527).
__global__ void __launch_bounds__(128) window_similarity_fc_kernel(const float* __restrict__ x, int D, int T, const float* __restrict__ wt /* [101][128] */,
                                                                   const float* __restrict__ bias, float* __restrict__ out, int out_ld, int out_coff) {
  extern __shared__ float sm[];
  float* xs = sm;       // [D]
  float* sims = sm + D; // [101]
  const int row = blockIdx.x, t = row % T, base = row - t, tid = threadIdx.x;
  for (int i = tid; i < D; i += 128) xs[i] = x[(long long)row * D + i];
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int j = warp; j < kLookup; j += 4) {
    const int t2 = t + j - (kLookup - 1) / 2;
    float s = 0.f;
    if (t2 >= 0 && t2 < T) {
      const float* y = x + (long long)(base + t2) * D;
      for (int i = lane; i < D; i += 32) s = fmaf(xs[i], y[i], s);
      for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    }
    if (lane == 0) sims[j] = s;
  }
  __syncthreads();
  float acc = bias[tid];
  for (int j = 0; j < kLookup; ++j) acc = fmaf(sims[j], wt[j * kSimDim + tid], acc);
  out[(long long)row * out_ld + out_coff + tid] = fmaxf(acc, 0.f);
}

// cls_layer1 + sigmoid (transnetv2.py:142-148): one warp per frame.  mode 0: prob[row]; mode 1 (video stitching,
// transnetv2_extraction_stages.py:258-263): frames 25..74 of window (w0 + b) land at 50 * (w0 + b) + t - 25 when < n.
__global__ void __launch_bounds__(128) head_kernel(const float* __restrict__ h, const float* __restrict__ w, float bias, int rows, int T, float* __restrict__ prob,
                                                   int stitch, int w0, int n_total) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s = 0.f;
  for (int i = lane; i < kFcOut; i += 32) s = fmaf(h[(long long)row * kFcOut + i], w[i], s);
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane) return;
  const float p = 1.0f / (1.0f + expf(-(s + bias)));
  if (!stitch) {
    prob[row] = p;
    return;
  }
  const int b = row / T, t = row % T;
  if (t < 25 || t >= 75) return;
  const long long dst = 50LL * (w0 + b) + t - 25;
  if (dst < n_total) prob[dst] = p;
}

struct TnBlock {
  int cin = 0, cin_pad = 0, filters = 0;
  bool relu = false;
  float *w1 = nullptr, *w2 = nullptr, *scale = nullptr, *shift = nullptr;  // device
};

}  // namespace cb

struct cb_transnet {
  cb_ctx* ctx = nullptr;
  std::map<std::string, std::vector<float>> host;  // tensors as uploaded (reference state_dict names)
  cb::TnBlock blk[cb::kStacks][cb::kBlocks];
  float *proj_wt = nullptr, *proj_b = nullptr, *sim_fc_wt = nullptr, *sim_fc_b = nullptr, *hist_fc_wt = nullptr, *hist_fc_b = nullptr;
  float *fc1_wt = nullptr, *fc1_b = nullptr, *cls_w = nullptr;
  float cls_b = 0.f;
  bool finalized = false;
  int max_windows = 0;
  // workspace for max_windows windows of <= 100 frames
  float *x0 = nullptr, *mid = nullptr, *b1 = nullptr, *b2 = nullptr, *p0 = nullptr, *p1 = nullptr, *hist = nullptr, *feats = nullptr, *proj = nullptr,
        *concat = nullptr, *fc1 = nullptr;
  int *d_first = nullptr, *d_pad = nullptr;
};

namespace cb {

static std::map<std::string, size_t> tn_expected() {
  std::map<std::string, size_t> e;
  for (int s = 0; s < kStacks; ++s) {
    const int f = 16 << s, stack_in = s == 0 ? 3 : (16 << (s - 1)) * 4;
    for (int b = 0; b < kBlocks; ++b) {
      const int cin = b == 0 ? stack_in : 4 * f;
      const std::string p = "SDDCNN." + std::to_string(s) + ".DDCNN." + std::to_string(b);
      for (int d : {1, 2, 4, 8}) {
        e[p + ".Conv3D_" + std::to_string(d) + ".layers.0.weight"] = (size_t)2 * f * cin * 9;
        e[p + ".Conv3D_" + std::to_string(d) + ".layers.1.weight"] = (size_t)f * 2 * f * 3;
      }
      for (const char* n : {"weight", "bias", "running_mean", "running_var"}) e[p + ".bn." + n] = (size_t)4 * f;
    }
  }
  e["frame_sim_layer.projection.weight"] = (size_t)kSimDim * 448, e["frame_sim_layer.projection.bias"] = kSimDim;
  e["frame_sim_layer.fc.weight"] = (size_t)kSimDim * kLookup, e["frame_sim_layer.fc.bias"] = kSimDim;
  e["color_hist_layer.fc.weight"] = (size_t)kSimDim * kLookup, e["color_hist_layer.fc.bias"] = kSimDim;
  e["fc1.weight"] = (size_t)kFcOut * kFcIn, e["fc1.bias"] = kFcOut;
  e["cls_layer1.weight"] = kFcOut, e["cls_layer1.bias"] = 1;
  return e;
}

static int upload(cb_ctx* ctx, float** dst, const std::vector<float>& v) {
  if (*dst) cudaFree(*dst), *dst = nullptr;
  CB_CUDA(ctx, cudaMalloc(dst, v.size() * sizeof(float)));
  CB_CUDA(ctx, cudaMemcpy(*dst, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
  return CB_OK;
}

// [out][in] Linear weight -> [in][out]
static std::vector<float> transposed(const std::vector<float>& w, int out, int in) {
  std::vector<float> t((size_t)in * out);
  for (int o = 0; o < out; ++o)
    for (int i = 0; i < in; ++i) t[(size_t)i * out + o] = w[(size_t)o * in + i];
  return t;
}

template <int CT, int TN, int BKC>
static int launch_conv(cb_ctx* ctx, const ConvGemmArgs& a, int zdim, cudaStream_t st) {
  constexpr int BM = 8 * 256 / CT, BN = CT * TN;
  dim3 grid((a.M + BM - 1) / BM, (a.N + BN - 1) / BN, zdim);
  mark_launch(ctx, CB_PROF_CONV, st);
  conv_gemm_kernel<CT, TN, BKC><<<grid, 256, 0, st>>>(a);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

static int conv_dispatch(cb_ctx* ctx, const ConvGemmArgs& a, int zdim, cudaStream_t st) {
  if (a.N % 4) return fail(ctx, CB_ERR_UNSUPPORTED, "transnet: N=%d is not a multiple of 4", a.N);
  if (a.cin % 16 == 0) {
    if (a.N >= 128) return launch_conv<16, 8, 16>(ctx, a, zdim, st);  // 128 x 128
    if (a.N >= 64) return launch_conv<8, 8, 16>(ctx, a, zdim, st);    // 256 x 64
    if (a.N >= 32) return launch_conv<8, 4, 16>(ctx, a, zdim, st);    // 256 x 32
    return launch_conv<4, 4, 8>(ctx, a, zdim, st);                    // 512 x 16
  }
  if (a.cin % 4 == 0 && a.N >= 128) return launch_conv<16, 8, 4>(ctx, a, zdim, st);
  return fail(ctx, CB_ERR_UNSUPPORTED, "transnet: no conv kernel for cin=%d N=%d", a.cin, a.N);
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }  // NULL counts as aligned

// One launch of conv_gemm_kernel over zdim branches.  Everything the float4 loads and stores need is checked here: the base
// pointers, and every row stride and column offset a multiple of 4 floats.  Modes 1 and 2 gather taps inside a frame (mode 1) or
// a window (mode 2), so M must hold whole frames, and for mode 2 whole windows: a tap of the last window would otherwise read rows
// past M.
static int conv(cb_ctx* ctx, const ConvGemmArgs& a, int zdim, cudaStream_t st) {
  if (!a.in || !a.w || !a.out) return fail(ctx, CB_ERR_ARG, "transnet conv: null operand");
  if (a.mode < 0 || a.mode > 2) return fail(ctx, CB_ERR_ARG, "transnet conv: mode=%d (0 rows, 1 spatial taps, 2 temporal taps)", a.mode);
  if (zdim < 1 || zdim > 65535) return fail(ctx, CB_ERR_ARG, "transnet conv: z=%d (1..65535)", zdim);
  if (a.M < 0 || a.N <= 0 || a.cin <= 0 || a.T <= 0 || a.H <= 0 || a.W <= 0 || a.dil < 0 || a.z_dil_shift < 0)
    return fail(ctx, CB_ERR_ARG, "transnet conv: M=%d N=%d cin=%d T=%d H=%d W=%d dil=%d", a.M, a.N, a.cin, a.T, a.H, a.W, a.dil);
  if (!aligned16(a.in) || !aligned16(a.w) || !aligned16(a.out) || ((uintptr_t)a.scale & 3) || ((uintptr_t)a.shift & 3))
    return fail(ctx, CB_ERR_ARG, "transnet conv: in, w and out must be 16-byte aligned, scale and shift 4-byte");
  if ((a.in_ld | a.in_coff | a.out_ld | a.out_coff | a.w_ld | a.z_in_coff | a.z_out_coff | (int)(a.z_w & 3)) & 3 || a.in_ld < 0 || a.in_coff < 0 ||
      a.out_ld < 0 || a.out_coff < 0 || a.w_ld < 0 || a.z_in_coff < 0 || a.z_out_coff < 0 || a.z_w < 0)
    return fail(ctx, CB_ERR_ARG, "transnet conv: in_ld=%d in_coff=%d out_ld=%d out_coff=%d w_ld=%d z_in_coff=%d z_out_coff=%d z_w=%lld must be multiples of 4",
                a.in_ld, a.in_coff, a.out_ld, a.out_coff, a.w_ld, a.z_in_coff, a.z_out_coff, a.z_w);
  const long long frame = (long long)a.H * a.W, rows_per_unit = a.mode == 2 ? frame * a.T : (a.mode == 1 ? frame : 1);
  if (a.M % rows_per_unit) return fail(ctx, CB_ERR_ARG, "transnet conv: M=%d is not a whole number of %s of %lld rows", a.M, a.mode == 2 ? "windows" : "frames", rows_per_unit);
  if (a.M == 0) return CB_OK;
  return conv_dispatch(ctx, a, zdim, st);
}

static int window_gather(cb_ctx* ctx, const uint8_t* frames, const int* first, const int* pad, int B, int T, float* x0, float* hist, cudaStream_t st) {
  if (!frames || !first || !pad || !x0 || !hist) return fail(ctx, CB_ERR_ARG, "transnet window_gather: null operand");
  if (B < 0 || T < 0 || (long long)B * T > INT32_MAX) return fail(ctx, CB_ERR_ARG, "transnet window_gather: B=%d T=%d", B, T);
  if (!aligned16(x0) || ((uintptr_t)first & 3) || ((uintptr_t)pad & 3) || ((uintptr_t)hist & 3))
    return fail(ctx, CB_ERR_ARG, "transnet window_gather: x0 must be 16-byte aligned, first, pad and hist 4-byte");
  if (B == 0 || T == 0) return CB_OK;
  mark_launch(ctx, CB_PROF_CONV, st);
  window_gather_kernel<<<B * T, 256, 0, st>>>(frames, first, pad, T, x0, hist);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

static int shortcut_pool(cb_ctx* ctx, const float* x2, const float* x1, float* out, int frames, int H, int W, int C, long long out_frame_stride, cudaStream_t st) {
  if (!x2 || !x1 || !out) return fail(ctx, CB_ERR_ARG, "transnet shortcut_pool: null operand");
  if (frames < 0 || H < 0 || W < 0 || C < 0 || out_frame_stride < 0)
    return fail(ctx, CB_ERR_ARG, "transnet shortcut_pool: frames=%d H=%d W=%d C=%d out_frame_stride=%lld", frames, H, W, C, out_frame_stride);
  if (!aligned16(x2) || !aligned16(x1) || !aligned16(out) || C % 4 || out_frame_stride % 4)
    return fail(ctx, CB_ERR_ARG, "transnet shortcut_pool: x2, x1, out must be 16-byte aligned, C=%d and out_frame_stride=%lld multiples of 4", C, out_frame_stride);
  const long long total = (long long)frames * (H / 2) * (W / 2) * (C / 4);
  if (total == 0) return CB_OK;
  const int blocks = (int)std::min<long long>((total + 255) / 256, 148LL * 16);
  mark_launch(ctx, CB_PROF_CONV, st);
  shortcut_pool_kernel<<<blocks, 256, 0, st>>>(x2, x1, out, frames, H, W, C, out_frame_stride);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

static int spatial_mean(cb_ctx* ctx, const float* x, long long frame_stride, int frames, int npos, int C, float* feats, int feats_ld, int coff, cudaStream_t st) {
  if (!x || !feats) return fail(ctx, CB_ERR_ARG, "transnet spatial_mean: null operand");
  if (frames < 0 || npos <= 0 || C < 0 || frame_stride < 0 || feats_ld < 0 || coff < 0)
    return fail(ctx, CB_ERR_ARG, "transnet spatial_mean: frames=%d npos=%d C=%d frame_stride=%lld feats_ld=%d coff=%d", frames, npos, C, frame_stride, feats_ld, coff);
  if (((uintptr_t)x & 3) || ((uintptr_t)feats & 3)) return fail(ctx, CB_ERR_ARG, "transnet spatial_mean: x and feats must be 4-byte aligned");
  if (frames == 0 || C == 0) return CB_OK;
  mark_launch(ctx, CB_PROF_CONV, st);
  spatial_mean_kernel<<<frames, 128, 0, st>>>(x, frame_stride, npos, C, feats, feats_ld, coff);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

static int l2_normalize_rows(cb_ctx* ctx, float* x, int rows, int D, cudaStream_t st) {
  if (!x) return fail(ctx, CB_ERR_ARG, "transnet l2_normalize_rows: null operand");
  if (rows < 0 || D <= 0) return fail(ctx, CB_ERR_ARG, "transnet l2_normalize_rows: rows=%d D=%d", rows, D);
  if ((uintptr_t)x & 3) return fail(ctx, CB_ERR_ARG, "transnet l2_normalize_rows: x must be 4-byte aligned");
  if (rows == 0) return CB_OK;
  mark_launch(ctx, CB_PROF_CONV, st);
  l2_normalize_rows_kernel<<<rows, 128, 0, st>>>(x, D);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

// rows = whole windows of T frames: every neighbour a row reads is a row of its own window.
static int window_similarity_fc(cb_ctx* ctx, const float* x, int rows, int D, int T, const float* wt, const float* bias, float* out, int out_ld, int out_coff,
                                cudaStream_t st) {
  if (!x || !wt || !bias || !out) return fail(ctx, CB_ERR_ARG, "transnet window_similarity_fc: null operand");
  if (rows < 0 || D <= 0 || T <= 0 || rows % T || out_ld < 0 || out_coff < 0)
    return fail(ctx, CB_ERR_ARG, "transnet window_similarity_fc: rows=%d D=%d T=%d out_ld=%d out_coff=%d (rows whole windows of T)", rows, D, T, out_ld, out_coff);
  if (((uintptr_t)x & 3) || ((uintptr_t)wt & 3) || ((uintptr_t)bias & 3) || ((uintptr_t)out & 3))
    return fail(ctx, CB_ERR_ARG, "transnet window_similarity_fc: operands must be 4-byte aligned");
  const size_t smem = ((size_t)D + kLookup) * sizeof(float);
  if (smem > 48 * 1024) return fail(ctx, CB_ERR_UNSUPPORTED, "transnet window_similarity_fc: D=%d: %zu bytes of shared memory exceed 48 KB", D, smem);
  if (rows == 0) return CB_OK;
  mark_launch(ctx, CB_PROF_CONV, st);
  window_similarity_fc_kernel<<<rows, 128, smem, st>>>(x, D, T, wt, bias, out, out_ld, out_coff);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

static int head(cb_ctx* ctx, const float* h, const float* w, float bias, int rows, int T, float* prob, int stitch, int w0, int n_total, cudaStream_t st) {
  if (!h || !w || !prob) return fail(ctx, CB_ERR_ARG, "transnet head: null operand");
  if (rows < 0 || T <= 0 || (stitch != 0 && stitch != 1) || w0 < 0 || n_total < 0)
    return fail(ctx, CB_ERR_ARG, "transnet head: rows=%d T=%d stitch=%d w0=%d n_total=%d", rows, T, stitch, w0, n_total);
  if (((uintptr_t)h & 3) || ((uintptr_t)w & 3) || ((uintptr_t)prob & 3)) return fail(ctx, CB_ERR_ARG, "transnet head: operands must be 4-byte aligned");
  if (rows == 0) return CB_OK;
  mark_launch(ctx, CB_PROF_CONV, st);
  head_kernel<<<(rows + 3) / 4, 128, 0, st>>>(h, w, bias, rows, T, prob, stitch, w0, n_total);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

// B windows of T frames each; window b = video frames first[b] + max(t - pad[b], 0).  prob: see head_kernel.
static int run_windows(cb_transnet* tn, const uint8_t* frames, const int* h_first, const int* h_pad, int B, int T, float* prob, int stitch, int w0, int n_total,
                       cudaStream_t st) {
  cb_ctx* ctx = tn->ctx;
  CB_CUDA(ctx, cudaMemcpyAsync(tn->d_first, h_first, B * sizeof(int), cudaMemcpyHostToDevice, st));
  CB_CUDA(ctx, cudaMemcpyAsync(tn->d_pad, h_pad, B * sizeof(int), cudaMemcpyHostToDevice, st));
  const int frames_n = B * T;
  int rc;
  if ((rc = window_gather(ctx, frames, tn->d_first, tn->d_pad, B, T, tn->x0, tn->hist, st))) return rc;

  int H = kFrameH, W = kFrameW;
  const float* x = tn->x0;
  int x_ld = 4;
  int feat_off = 0;
  for (int s = 0; s < kStacks; ++s) {
    const int f = 16 << s, C = 4 * f, M = frames_n * H * W;
    float* outs[2] = {tn->b1, tn->b2};
    for (int b = 0; b < kBlocks; ++b) {
      const TnBlock& k = tn->blk[s][b];
      ConvGemmArgs a{};
      a.in = x, a.w = k.w1, a.out = tn->mid, a.scale = nullptr, a.shift = nullptr;
      a.M = M, a.N = 8 * f, a.cin = k.cin_pad, a.in_ld = x_ld, a.in_coff = 0, a.w_ld = 8 * f, a.out_ld = 8 * f, a.out_coff = 0;
      a.T = T, a.H = H, a.W = W, a.mode = 1, a.dil = 1, a.relu = 0;
      if ((rc = conv(ctx, a, 1, st))) return rc;
      ConvGemmArgs t{};
      t.in = tn->mid, t.w = k.w2, t.out = outs[b], t.scale = k.scale, t.shift = k.shift;
      t.M = M, t.N = f, t.cin = 2 * f, t.in_ld = 8 * f, t.in_coff = 0, t.w_ld = f, t.out_ld = C, t.out_coff = 0;
      t.T = T, t.H = H, t.W = W, t.mode = 2, t.relu = k.relu ? 1 : 0;
      t.z_in_coff = 2 * f, t.z_out_coff = f, t.z_w = (long long)3 * 2 * f * f;
      t.dil = 1, t.z_dil_shift = 1;  // branch z: dilation 1 << z, its own channel slices and weights
      if ((rc = conv(ctx, t, kBranches, st))) return rc;
      x = outs[b], x_ld = C;
    }
    const int Hp = H / 2, Wp = W / 2;
    float* pooled = s == 0 ? tn->p0 : (s == 1 ? tn->p1 : tn->concat + kTrunkOff);
    const long long fstride = s == 2 ? kFcIn : (long long)Hp * Wp * C;
    if ((rc = shortcut_pool(ctx, tn->b2, tn->b1, pooled, frames_n, H, W, C, fstride, st))) return rc;
    if ((rc = spatial_mean(ctx, pooled, fstride, frames_n, Hp * Wp, C, tn->feats, 448, feat_off, st))) return rc;
    feat_off += C;
    x = pooled, x_ld = C, H = Hp, W = Wp;
  }
  // learned frame similarity
  {
    ConvGemmArgs a{};
    a.in = tn->feats, a.w = tn->proj_wt, a.out = tn->proj, a.shift = tn->proj_b;
    a.M = frames_n, a.N = kSimDim, a.cin = 448, a.in_ld = 448, a.w_ld = kSimDim, a.out_ld = kSimDim;
    a.T = T, a.H = 1, a.W = 1, a.mode = 0;
    if ((rc = conv(ctx, a, 1, st))) return rc;
    if ((rc = l2_normalize_rows(ctx, tn->proj, frames_n, kSimDim, st))) return rc;
    if ((rc = window_similarity_fc(ctx, tn->proj, frames_n, kSimDim, T, tn->sim_fc_wt, tn->sim_fc_b, tn->concat, kFcIn, kSimDim, st))) return rc;
    if ((rc = window_similarity_fc(ctx, tn->hist, frames_n, kHistBins, T, tn->hist_fc_wt, tn->hist_fc_b, tn->concat, kFcIn, 0, st))) return rc;
  }
  {
    ConvGemmArgs a{};
    a.in = tn->concat, a.w = tn->fc1_wt, a.out = tn->fc1, a.shift = tn->fc1_b;
    a.M = frames_n, a.N = kFcOut, a.cin = kFcIn, a.in_ld = kFcIn, a.w_ld = kFcOut, a.out_ld = kFcOut;
    a.T = T, a.H = 1, a.W = 1, a.mode = 0, a.relu = 1;
    if ((rc = conv(ctx, a, 1, st))) return rc;
    if ((rc = head(ctx, tn->fc1, tn->cls_w, tn->cls_b, frames_n, T, prob, stitch, w0, n_total, st))) return rc;
  }
  return CB_OK;
}

static void free_workspace(cb_transnet* tn) {
  for (float** p : {&tn->x0, &tn->mid, &tn->b1, &tn->b2, &tn->p0, &tn->p1, &tn->hist, &tn->feats, &tn->proj, &tn->concat, &tn->fc1})
    if (*p) cudaFree(*p), *p = nullptr;
  if (tn->d_first) cudaFree(tn->d_first), tn->d_first = nullptr;
  if (tn->d_pad) cudaFree(tn->d_pad), tn->d_pad = nullptr;
}

}  // namespace cb

extern "C" {

int cb_transnet_create(cb_ctx* ctx, cb_transnet** out) {
  if (!ctx) return CB_ERR_ARG;
  if (!out) return cb::fail(ctx, CB_ERR_ARG, "transnet_create: null argument");
  cb_transnet* tn = new cb_transnet();
  tn->ctx = ctx;
  *out = tn;
  return CB_OK;
}

void cb_transnet_destroy(cb_transnet* tn) {
  if (!tn) return;
  cudaSetDevice(tn->ctx->device);
  cb::free_workspace(tn);
  for (auto& st : tn->blk)
    for (auto& k : st) cudaFree(k.w1), cudaFree(k.w2), cudaFree(k.scale), cudaFree(k.shift);
  for (float* p : {tn->proj_wt, tn->proj_b, tn->sim_fc_wt, tn->sim_fc_b, tn->hist_fc_wt, tn->hist_fc_b, tn->fc1_wt, tn->fc1_b, tn->cls_w}) cudaFree(p);
  delete tn;
}

int cb_transnet_set_tensor(cb_transnet* tn, const char* name, const float* data, size_t count) {
  if (!tn) return CB_ERR_ARG;
  cb_ctx* ctx = tn->ctx;
  if (!name || !data) return cb::fail(ctx, CB_ERR_ARG, "transnet_set_tensor: null argument");
  static const std::map<std::string, size_t> exp = cb::tn_expected();
  auto it = exp.find(name);
  if (it == exp.end()) return cb::fail(ctx, CB_ERR_ARG, "transnet_set_tensor: unknown tensor '%s'", name);
  if (it->second != count) return cb::fail(ctx, CB_ERR_ARG, "transnet_set_tensor: '%s' has %zu elements, expected %zu", name, count, it->second);
  tn->host[name].assign(data, data + count);
  tn->finalized = false;
  return CB_OK;
}

int cb_transnet_finalize(cb_transnet* tn, int max_windows) {
  if (!tn) return CB_ERR_ARG;
  cb_ctx* ctx = tn->ctx;
  if (max_windows <= 0 || max_windows > 256) return cb::fail(ctx, CB_ERR_ARG, "transnet_finalize: max_windows must be in 1..256");
  for (auto& kv : cb::tn_expected())
    if (!tn->host.count(kv.first)) return cb::fail(ctx, CB_ERR_STATE, "transnet_finalize: tensor '%s' was never set", kv.first.c_str());
  CB_CUDA(ctx, cudaSetDevice(ctx->device));
  int rc;
  for (int s = 0; s < cb::kStacks; ++s) {
    const int f = 16 << s, stack_in = s == 0 ? 3 : (16 << (s - 1)) * 4;
    for (int b = 0; b < cb::kBlocks; ++b) {
      cb::TnBlock& k = tn->blk[s][b];
      k.cin = b == 0 ? stack_in : 4 * f, k.cin_pad = (k.cin + 3) & ~3, k.filters = f, k.relu = b != cb::kBlocks - 1;
      const std::string p = "SDDCNN." + std::to_string(s) + ".DDCNN." + std::to_string(b);
      // (1,3,3) convs of the four branches side by side: Wt[(tap*cin_pad + ci)][branch*2F + co]
      std::vector<float> w1((size_t)9 * k.cin_pad * 8 * f, 0.f), w2((size_t)4 * 3 * 2 * f * f);
      for (int br = 0; br < 4; ++br) {
        const std::string c = p + ".Conv3D_" + std::to_string(1 << br) + ".layers.";
        const std::vector<float>& a = tn->host[c + "0.weight"];  // [2F][cin][1][3][3]
        for (int co = 0; co < 2 * f; ++co)
          for (int ci = 0; ci < k.cin; ++ci)
            for (int tap = 0; tap < 9; ++tap) w1[((size_t)tap * k.cin_pad + ci) * 8 * f + br * 2 * f + co] = a[((size_t)co * k.cin + ci) * 9 + tap];
        const std::vector<float>& t = tn->host[c + "1.weight"];  // [F][2F][3][1][1]
        for (int fo = 0; fo < f; ++fo)
          for (int c2 = 0; c2 < 2 * f; ++c2)
            for (int kt = 0; kt < 3; ++kt) w2[(size_t)br * 3 * 2 * f * f + ((size_t)kt * 2 * f + c2) * f + fo] = t[((size_t)fo * 2 * f + c2) * 3 + kt];
      }
      // BatchNorm3d(eps=1e-3) in eval mode: y = (x - mean) / sqrt(var + eps) * gamma + beta  ->  x * scale + shift
      std::vector<float> sc(4 * f), sh(4 * f);
      const auto &g = tn->host[p + ".bn.weight"], &be = tn->host[p + ".bn.bias"], &mu = tn->host[p + ".bn.running_mean"], &var = tn->host[p + ".bn.running_var"];
      for (int c = 0; c < 4 * f; ++c) {
        const double inv = 1.0 / std::sqrt((double)var[c] + 1e-3);
        sc[c] = (float)((double)g[c] * inv);
        sh[c] = (float)((double)be[c] - (double)mu[c] * (double)g[c] * inv);
      }
      if ((rc = cb::upload(ctx, &k.w1, w1)) || (rc = cb::upload(ctx, &k.w2, w2)) || (rc = cb::upload(ctx, &k.scale, sc)) || (rc = cb::upload(ctx, &k.shift, sh)))
        return rc;
    }
  }
  if ((rc = cb::upload(ctx, &tn->proj_wt, cb::transposed(tn->host["frame_sim_layer.projection.weight"], cb::kSimDim, 448)))) return rc;
  if ((rc = cb::upload(ctx, &tn->proj_b, tn->host["frame_sim_layer.projection.bias"]))) return rc;
  if ((rc = cb::upload(ctx, &tn->sim_fc_wt, cb::transposed(tn->host["frame_sim_layer.fc.weight"], cb::kSimDim, cb::kLookup)))) return rc;
  if ((rc = cb::upload(ctx, &tn->sim_fc_b, tn->host["frame_sim_layer.fc.bias"]))) return rc;
  if ((rc = cb::upload(ctx, &tn->hist_fc_wt, cb::transposed(tn->host["color_hist_layer.fc.weight"], cb::kSimDim, cb::kLookup)))) return rc;
  if ((rc = cb::upload(ctx, &tn->hist_fc_b, tn->host["color_hist_layer.fc.bias"]))) return rc;
  if ((rc = cb::upload(ctx, &tn->fc1_wt, cb::transposed(tn->host["fc1.weight"], cb::kFcOut, cb::kFcIn)))) return rc;
  if ((rc = cb::upload(ctx, &tn->fc1_b, tn->host["fc1.bias"]))) return rc;
  if ((rc = cb::upload(ctx, &tn->cls_w, tn->host["cls_layer1.weight"]))) return rc;
  tn->cls_b = tn->host["cls_layer1.bias"][0];

  cb::free_workspace(tn);
  const size_t fr = (size_t)max_windows * 100, pos0 = fr * cb::kFrameH * cb::kFrameW;
  auto alloc = [&](float** p, size_t n) -> int {
    CB_CUDA(ctx, cudaMalloc(p, n * sizeof(float)));
    return CB_OK;
  };
  if ((rc = alloc(&tn->x0, pos0 * 4)) || (rc = alloc(&tn->mid, pos0 * 128)) || (rc = alloc(&tn->b1, pos0 * 64)) || (rc = alloc(&tn->b2, pos0 * 64)) ||
      (rc = alloc(&tn->p0, fr * 13 * 24 * 64)) || (rc = alloc(&tn->p1, fr * 6 * 12 * 128)) || (rc = alloc(&tn->hist, fr * cb::kHistBins)) ||
      (rc = alloc(&tn->feats, fr * 448)) || (rc = alloc(&tn->proj, fr * cb::kSimDim)) || (rc = alloc(&tn->concat, fr * cb::kFcIn)) ||
      (rc = alloc(&tn->fc1, fr * cb::kFcOut)))
    return rc;
  CB_CUDA(ctx, cudaMalloc(&tn->d_first, max_windows * sizeof(int)));
  CB_CUDA(ctx, cudaMalloc(&tn->d_pad, max_windows * sizeof(int)));
  tn->max_windows = max_windows;
  tn->finalized = true;
  return CB_OK;
}

int cb_transnet_forward(cb_transnet* tn, const uint8_t* windows, int n_windows, int frames_per_window, float* prob_out, void* stream) {
  if (!tn) return CB_ERR_ARG;
  cb_ctx* ctx = tn->ctx;
  if (!tn->finalized) return cb::fail(ctx, CB_ERR_STATE, "transnet_forward: call cb_transnet_finalize first");
  if (!windows || !prob_out || n_windows <= 0) return cb::fail(ctx, CB_ERR_ARG, "transnet_forward: null/empty argument");
  if (frames_per_window <= 0 || frames_per_window > 100) return cb::fail(ctx, CB_ERR_ARG, "transnet_forward: 1..100 frames per window, got %d", frames_per_window);
  CB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int T = frames_per_window;
  std::vector<int> first, pad;
  for (int w = 0; w < n_windows; w += tn->max_windows) {
    const int B = std::min(tn->max_windows, n_windows - w);
    first.resize(B), pad.assign(B, 0);
    for (int b = 0; b < B; ++b) first[b] = (w + b) * T;
    // the index arrays are copied with cudaMemcpyAsync from pageable memory: staged before the call returns
    int rc = cb::run_windows(tn, windows, first.data(), pad.data(), B, T, prob_out + (size_t)w * T, 0, 0, 0, st);
    if (rc) return rc;
  }
  return CB_OK;
}

int cb_transnet_predict(cb_transnet* tn, const uint8_t* frames, int n_frames, float* prob_out, void* stream) {
  if (!tn) return CB_ERR_ARG;
  cb_ctx* ctx = tn->ctx;
  if (!tn->finalized) return cb::fail(ctx, CB_ERR_STATE, "transnet_predict: call cb_transnet_finalize first");
  if (!frames || !prob_out || n_frames <= 0) return cb::fail(ctx, CB_ERR_ARG, "transnet_predict: null/empty argument");
  CB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  // window plan of _get_batches (transnetv2_extraction_stages.py:215-236): window i covers video frames
  // [max(50i-25,0), min(50i+75,n)), front-padded with frame 0 to start at 50i-25; the END is never padded.
  const int rem = (50 - n_frames % 50) % 50, n_win = (n_frames + rem) / 50;
  std::vector<int> first, pad;
  int w = 0;
  while (w < n_win) {
    auto len_of = [&](int i) { return std::min(50 * i + 75, n_frames) - std::max(50 * i - 25, 0) + std::max(25 - 50 * i, 0); };
    const int T = len_of(w);
    int B = 1;
    while (w + B < n_win && B < tn->max_windows && len_of(w + B) == T) ++B;
    first.resize(B), pad.resize(B);
    for (int b = 0; b < B; ++b) first[b] = std::max(50 * (w + b) - 25, 0), pad[b] = std::max(25 - 50 * (w + b), 0);
    int rc = cb::run_windows(tn, frames, first.data(), pad.data(), B, T, prob_out, 1, w, n_frames, st);
    if (rc) return rc;
    w += B;
  }
  return CB_OK;
}

int cb_transnet_conv(cb_ctx* ctx, const cb_transnet_conv_args* a, int z, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  if (!a) return cb::fail(ctx, CB_ERR_ARG, "transnet conv: null argument");
  cb::ConvGemmArgs g{};
  g.in = a->in, g.w = a->w, g.out = a->out, g.scale = a->scale, g.shift = a->shift;
  g.M = a->M, g.N = a->N, g.cin = a->cin, g.in_ld = a->in_ld, g.in_coff = a->in_coff, g.w_ld = a->w_ld, g.out_ld = a->out_ld, g.out_coff = a->out_coff;
  g.T = a->T, g.H = a->H, g.W = a->W, g.mode = a->mode, g.dil = a->dil, g.relu = a->relu;
  g.z_in_coff = a->z_in_coff, g.z_out_coff = a->z_out_coff, g.z_dil_shift = a->z_dil_shift, g.z_w = a->z_w;
  return cb::conv(ctx, g, z, (cudaStream_t)stream);
}

int cb_transnet_window_gather(cb_ctx* ctx, const uint8_t* frames, const int32_t* first, const int32_t* pad, int B, int T, float* x0, float* hist, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::window_gather(ctx, frames, first, pad, B, T, x0, hist, (cudaStream_t)stream);
}

int cb_transnet_shortcut_pool(cb_ctx* ctx, const float* x2, const float* x1, float* out, int frames, int H, int W, int C, long long out_frame_stride, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::shortcut_pool(ctx, x2, x1, out, frames, H, W, C, out_frame_stride, (cudaStream_t)stream);
}

int cb_transnet_spatial_mean(cb_ctx* ctx, const float* x, long long frame_stride, int frames, int npos, int C, float* feats, int feats_ld, int coff, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::spatial_mean(ctx, x, frame_stride, frames, npos, C, feats, feats_ld, coff, (cudaStream_t)stream);
}

int cb_transnet_l2_normalize_rows(cb_ctx* ctx, float* x, int rows, int D, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::l2_normalize_rows(ctx, x, rows, D, (cudaStream_t)stream);
}

int cb_transnet_window_similarity_fc(cb_ctx* ctx, const float* x, int rows, int D, int T, const float* wt, const float* bias, float* out, int out_ld, int out_coff,
                                     void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::window_similarity_fc(ctx, x, rows, D, T, wt, bias, out, out_ld, out_coff, (cudaStream_t)stream);
}

int cb_transnet_head(cb_ctx* ctx, const float* h, const float* w, float bias, int rows, int T, float* prob, int stitch, int w0, int n_total, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::head(ctx, h, w, bias, rows, T, prob, stitch, w0, n_total, (cudaStream_t)stream);
}

}  // extern "C"
