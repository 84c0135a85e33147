// wgmma GEMM for the image tower (sm_90a):  C[M][N] = epilogue(A[M][K] . W[N][K]^T + bias) (+ residual)
//
//  * fp16 operands, fp32 accumulation in registers; one 128 x BN output tile per CTA iteration, persistent grid (one CTA
//    per SM) walking tiles n-fastest so the A row-block stays in L2 while W streams.
//  * warpgroup 0: warp 0 is the TMA producer (cp.async.bulk.tensor 2-D, 128-byte swizzle, kStages-deep mbarrier ring); the
//    group gives its registers away (setmaxnreg).
//    warpgroups 1-2: consumers; each owns 64 rows of the tile (wgmma m64 x BN x k16, both operands from shared memory), keeps
//    one k-block of MMAs in flight and runs the epilogue (bias / activation / residual) from its accumulator registers.
//  * Epilogue: each consumer warpgroup writes its 64 rows in column slices of 128 bytes (32 fp32 / 64 fp16 columns, 8 KB, in
//    TMA's 128-byte swizzle, which also keeps the shared-memory writes free of bank conflicts) into two buffers of its own; a
//    TMA store takes each slice to global memory while the warpgroup goes on, and clips the rows / columns past M / N. The
//    tile's bias is read once, into registers, while its last MMAs run; no other global access sits on the consumers' path.
//    With a residual, its slices arrive by TMA load into the same buffers (the first two during the tile's mainloop, the
//    rest as buffers free up; the producer prefetches the whole residual tile into L2 when it starts the tile), the epilogue
//    adds into them and the store writes them back. `residual` may alias the output: every tile reads its own region before
//    it writes it, and tiles are disjoint.
//  * Every Linear of HF CLIPEncoderLayer / SiglipEncoderLayer (q,k,v fused; out_proj; fc1; fc2) and the patch-embed conv
//    (im2col rows produced by the preprocess kernel) go through this kernel.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>

#include "common.h"
#include "ptx.cuh"

namespace cb {

constexpr int BM = 128, BK = 64;
constexpr int kGemmThreads = 384;
constexpr int kEpiRows = 64, kEpiBytes = kEpiRows * 128;  // one epilogue slice: a consumer warpgroup's 64 rows x 128 bytes

template <int BN>
struct GemmCfg {
  static constexpr int kStages = (BN == 256) ? 4 : 6;
  static constexpr int kABytes = BM * BK * 2, kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRingBytes = kStages * kStageBytes;
  static constexpr int kEpiTotal = 2 /*consumer warpgroups*/ * 2 /*buffers*/ * kEpiBytes;
  static constexpr int kSmem = kRingBytes + kEpiTotal + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmem <= 232448, "over the 227 KB of opt-in shared memory per block on sm_90");
};

struct GemmArgs {
  const float* bias;  // [N] or null
  int M, N, K;
  int residual;  // nonzero: add the [M][N] fp32 tensor of map_r (fp32 output only)
  const float* gamma;  // [N] per-column scale of (acc + bias), applied before the residual add (SCALE instantiations only)
};

// x * sigmoid(1.702 x) with one ex2.approx + one rcp.approx (both ~1 ulp; the result is rounded to fp16 anyway)
__device__ __forceinline__ float act_quick_gelu(float x) { return __fdividef(x, 1.f + exp2f(-2.4554669595930156f * x)); }
__device__ __forceinline__ float act_gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  const float e = exp2f(2.885390081777927f * u);  // e^{2u}; tanh(u) = 1 - 2/(e^{2u}+1)
  const float t = 1.f - __fdividef(2.f, e + 1.f);
  return 0.5f * x * (1.f + t);
}

// nn.GELU(): 0.5 x (1 + erf(x / sqrt(2))); CUDA's erff is within 2 ulp
__device__ __forceinline__ float act_gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }

template <int ACT>
__device__ __forceinline__ float act(float x) {
  if (ACT == CB_EPI_QUICK_GELU) return act_quick_gelu(x);
  if (ACT == CB_EPI_GELU_TANH) return act_gelu_tanh(x);
  if (ACT == CB_EPI_GELU_ERF) return act_gelu_erf(x);
  return x;
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db, int accumulate) {
  if (BN == 256) wgmma_m64n256k16(d, da, db, accumulate);
  else wgmma_m64n128k16(d, da, db, accumulate);
}

// map_o: the output ([M][N] fp32 or fp16, box 128 bytes x 64 rows, 128-byte swizzle); map_r: the residual, same box (read only
// when g.residual is set).  SCALE (fp32 output only): out = residual + gamma * (acc + bias), LayerScale; gamma is read once per
// tile beside the bias.
template <int BN, int ACT, bool OUT_F32, bool SCALE = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
    gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_o,
                      const __grid_constant__ CUtensorMap map_r, const GemmArgs g) {
  using Cfg = GemmCfg<BN>;
  constexpr int kSliceCols = OUT_F32 ? 32 : 64;  // columns per 128-byte slice row
  constexpr int kSlices = BN / kSliceCols;
  constexpr int kSliceJ = kSliceCols / 8;  // 8-column accumulator blocks per slice
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - smem_u32(smem_raw));
  uint8_t* sA = smem;                                // [stages][128][64] fp16, SW128
  uint8_t* sB = smem + Cfg::kStages * Cfg::kABytes;  // [stages][BN][64]
  uint8_t* sE = smem + Cfg::kRingBytes;              // [consumer warpgroup][2][64][128 B], SW128
  uint64_t* full = (uint64_t*)(smem + Cfg::kRingBytes + Cfg::kEpiTotal);
  uint64_t* empty = full + Cfg::kStages;
  uint64_t* rfull = empty + Cfg::kStages;  // [consumer warpgroup][2]: residual slice landed in that buffer

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int m_tiles = (g.M + BM - 1) / BM, n_tiles = (g.N + BN - 1) / BN;
  const int num_tiles = m_tiles * n_tiles;
  const int num_kb = (g.K + BK - 1) / BK;
  const int first = blockIdx.x, step = gridDim.x;
  const bool has_res = OUT_F32 && g.residual;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_o);
    if (has_res) tma_prefetch_desc(&map_r);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    for (int i = 0; i < 4; ++i) mbar_init(&rfull[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (warp == 0 && lane == 0) {  // ===== TMA producer
      int stage = 0;
      uint32_t phase = 0;
      for (int t = first; t < num_tiles; t += step) {
        const int m_blk = t / n_tiles, n_blk = t % n_tiles;
        if (has_res)  // the consumers' residual loads of this tile then hit L2
          for (int r = 0; r < BM; r += kEpiRows)
            for (int cc = 0; cc < BN && n_blk * BN + cc < g.N; cc += kSliceCols) tma_prefetch_l2_2d(&map_r, n_blk * BN + cc, m_blk * BM + r);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], Cfg::kStageBytes);
          tma_load_2d(sA + stage * Cfg::kABytes, &map_a, &full[stage], kb * BK, m_blk * BM);
          tma_load_2d(sB + stage * Cfg::kBBytes, &map_b, &full[stage], kb * BK, n_blk * BN);
          if (++stage == Cfg::kStages) stage = 0, phase ^= 1;
        }
      }
    }
  } else {  // ===== consumers: warpgroup c owns rows 64c..64c+63 of the tile
    reg_alloc<232>();
    const int c = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;  // issues and waits for this warpgroup's TMA stores / residual loads
    auto release = [&](int s) {  // this warpgroup's MMAs have finished reading slot s
      if (leader) mbar_arrive(&empty[s]);
    };
    uint8_t* ebuf = sE + c * 2 * kEpiBytes;
    uint64_t* rbar = rfull + 2 * c;
    int eb = 0;           // buffer of the next slice (alternates across slices and tiles)
    uint32_t rphase = 0;  // bit b: parity of rbar[b]'s next completion
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    float2 bias[BN / 8];
    float2 gam[SCALE ? BN / 8 : 1];
    for (int t = first; t < num_tiles; t += step) {
      const int m_blk = t / n_tiles, n_blk = t % n_tiles;
      const int row0 = m_blk * BM + c * 64, col0 = n_blk * BN;
      // slices holding in-range columns; none when all 64 rows are past M (the M tail)
      const int nslices = row0 >= g.M ? 0 : std::min(kSlices, (g.N - col0 + kSliceCols - 1) / kSliceCols);
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t da = wgmma_desc_sw128(smem_u32(sA + stage * Cfg::kABytes + c * (64 * 128)));
        const uint64_t db = wgmma_desc_sw128(smem_u32(sB + stage * Cfg::kBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_tile<BN>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) != 0);
        wgmma_commit();
        if (kb == 0 && has_res && leader) {  // the first two residual slices of the tile, while its MMAs run
          bulk_wait_read<0>();               // the previous tile's stores have left both buffers
          for (int s = 0; s < 2 && s < nslices; ++s) {
            const int b = eb ^ s;
            mbar_expect_tx(&rbar[b], kEpiBytes);
            tma_load_2d(ebuf + b * kEpiBytes, &map_r, &rbar[b], col0 + s * kSliceCols, row0);
          }
        }
        wgmma_wait<1>();  // the previous k-block's MMAs are complete: its slot may be refilled
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == Cfg::kStages) stage = 0, phase ^= 1;
      }
      // the tile's bias pairs: bias[j] = columns 8j + 2(lane%4) + 0..1 (N is a multiple of 8: a pair is in range or not as a whole)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col0 + 8 * j + 2 * (lane & 3);
        bias[j] = (g.bias && col < g.N) ? __ldg((const float2*)(g.bias + col)) : make_float2(0.f, 0.f);
        if (SCALE) gam[j] = col < g.N ? __ldg((const float2*)(g.gamma + col)) : make_float2(0.f, 0.f);
      }
      wgmma_wait<0>();
      release(prev);

      // epilogue: acc[4j + 0..1] = (local row rl, columns 8j + 2(lane%4) + 0..1), acc[4j + 2..3] = row rl + 8. In the
      // swizzled slice, the 16-byte chunk q of row r sits at chunk q ^ (r % 8), and r % 8 = lane / 4 for both rows.
      const int rl = (warp & 3) * 16 + (lane >> 2), sw = lane >> 2;
#pragma unroll
      for (int s = 0; s < kSlices; ++s) {
        if (s >= nslices) break;
        uint8_t* buf = ebuf + eb * kEpiBytes;
        if (has_res) {
          mbar_wait(&rbar[eb], (rphase >> eb) & 1);
          rphase ^= 1u << eb;
        } else {
          if (leader) bulk_wait_read<1>();  // the store issued from this buffer two slices ago has read it
          named_bar_sync(1 + c, 128);
        }
#pragma unroll
        for (int jj = 0; jj < kSliceJ; ++jj) {
          const int j = s * kSliceJ + jj;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint8_t* row = buf + (rl + 8 * h) * 128;
            float v0 = act<ACT>(acc[4 * j + 2 * h] + bias[j].x), v1 = act<ACT>(acc[4 * j + 2 * h + 1] + bias[j].y);
            // LayerScale as its own rounded product (the reference's x + gamma * y in fp32): left contractible, the compiler fuses it
            // into the residual add in some unrolled copies and not others, and a row's result would depend on its slot in the tile
            if (SCALE) v0 = __fmul_rn(v0, gam[j].x), v1 = __fmul_rn(v1, gam[j].y);
            if (OUT_F32) {
              float2* p = (float2*)(row + (((2 * jj + ((lane & 3) >> 1)) ^ sw) << 4) + 8 * (lane & 1));
              if (has_res) {
                const float2 rr = *p;
                v0 += rr.x, v1 += rr.y;
              }
              *p = make_float2(v0, v1);
            } else {
              *(__half2*)(row + ((jj ^ sw) << 4) + 4 * (lane & 3)) = __floats2half2_rn(v0, v1);
            }
          }
        }
        fence_proxy_async();  // this thread's writes are visible to the TMA store
        named_bar_sync(1 + c, 128);
        if (leader) {
          tma_store_2d(&map_o, buf, col0 + s * kSliceCols, row0);
          bulk_commit();
          if (has_res && s + 2 < nslices) {  // refill this buffer with the residual two slices on
            bulk_wait_read<0>();
            mbar_expect_tx(&rbar[eb], kEpiBytes);
            tma_load_2d(buf, &map_r, &rbar[eb], col0 + (s + 2) * kSliceCols, row0);
          }
        }
        eb ^= 1;
      }
    }
    if (leader) bulk_wait<0>();  // the stores are complete before the CTA's shared memory goes away
  }
}

template <int BN, int ACT, bool OUT_F32, bool SCALE = false>
static int launch_gemm(cb_ctx* ctx, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr, const GemmArgs& g,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_wgmma_kernel<BN, ACT, OUT_F32, SCALE>;
  static bool attr_done[64] = {};  // per template instantiation AND per device
  bool& attr_set = attr_done[ctx->device & 63];
  if (!attr_set) {
    CB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    attr_set = true;
  }
  const int tiles = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
  mark_launch(ctx, CB_PROF_GEMM, stream);
  kern<<<std::min(tiles, ctx->sm_count), kGemmThreads, Cfg::kSmem, stream>>>(ma, mb, mo, mr, g);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

template <int BN>
static int dispatch_gemm(cb_ctx* ctx, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr, const GemmArgs& g,
                         bool out_f32, int epilogue, cudaStream_t stream) {
  if (out_f32) return launch_gemm<BN, CB_EPI_NONE, true>(ctx, ma, mb, mo, mr, g, stream);
  if (epilogue == CB_EPI_QUICK_GELU) return launch_gemm<BN, CB_EPI_QUICK_GELU, false>(ctx, ma, mb, mo, mr, g, stream);
  if (epilogue == CB_EPI_GELU_TANH) return launch_gemm<BN, CB_EPI_GELU_TANH, false>(ctx, ma, mb, mo, mr, g, stream);
  if (epilogue == CB_EPI_GELU_ERF) return launch_gemm<BN, CB_EPI_GELU_ERF, false>(ctx, ma, mb, mo, mr, g, stream);
  if (epilogue == CB_EPI_NONE) return launch_gemm<BN, CB_EPI_NONE, false>(ctx, ma, mb, mo, mr, g, stream);
  return fail(ctx, CB_ERR_ARG, "gemm: unknown epilogue %d", epilogue);
}

// gamma: nullable [N] LayerScale (fp32 output only); its tiles are 128 x 128 (the scale's registers sit beside the bias')
int gemm_f16_ex(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* gamma, const float* residual, float* out_f32,
                void* out_f16, int M, int N, int K, int epilogue, cudaStream_t stream) {
  if (!A || !W || (!out_f32 && !out_f16)) return fail(ctx, CB_ERR_ARG, "gemm: null operand");
  if (M <= 0 || N <= 0 || K <= 0) return fail(ctx, CB_ERR_ARG, "gemm: bad shape %dx%dx%d", M, N, K);
  if ((K & 7) || (N & 7)) return fail(ctx, CB_ERR_ARG, "gemm: N and K must be multiples of 8 (got N=%d K=%d)", N, K);
  if (((uintptr_t)A | (uintptr_t)W) & 15) return fail(ctx, CB_ERR_ARG, "gemm: operands must be 16-byte aligned");
  const void* out = out_f32 ? (const void*)out_f32 : out_f16;
  if (((uintptr_t)out | (uintptr_t)residual) & 15) return fail(ctx, CB_ERR_ARG, "gemm: output and residual must be 16-byte aligned");
  if (out_f32 && epilogue != CB_EPI_NONE) return fail(ctx, CB_ERR_UNSUPPORTED, "gemm: activation with fp32 output");
  if (residual && !out_f32) return fail(ctx, CB_ERR_UNSUPPORTED, "gemm: residual needs the fp32 output");
  if (gamma && !out_f32) return fail(ctx, CB_ERR_UNSUPPORTED, "gemm: gamma needs the fp32 output");
  if ((uintptr_t)gamma & 7) return fail(ctx, CB_ERR_ARG, "gemm: gamma must be 8-byte aligned");
  // 128 x 256 tiles when that still fills the machine, else 128 x 128
  const int tiles256 = ((M + BM - 1) / BM) * ((N + 255) / 256);
  const bool wide = !gamma && (N % 256 == 0 || N > 1024) && tiles256 >= ctx->sm_count;
  const int BN = wide ? 256 : 128;
  CUtensorMap ma, mb, mo, mr;
  uint64_t da[2] = {(uint64_t)K, (uint64_t)M}, db[2] = {(uint64_t)K, (uint64_t)N}, st[1] = {(uint64_t)K * 2};
  uint32_t ba[2] = {BK, BM}, bb[2] = {BK, (uint32_t)BN};
  int rc = make_tensor_map(ctx, &ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, A, da, st, ba, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  rc = make_tensor_map(ctx, &mb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W, db, st, bb, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  // output / residual: boxes of 64 rows x 128 bytes, the epilogue's slices
  const uint64_t esz = out_f32 ? 4 : 2;
  uint64_t dout[2] = {(uint64_t)N, (uint64_t)M}, sout[1] = {(uint64_t)N * esz};
  uint32_t bout[2] = {(uint32_t)(128 / esz), (uint32_t)kEpiRows};
  const CUtensorMapDataType dt = out_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  rc = make_tensor_map(ctx, &mo, dt, 2, out, dout, sout, bout, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  mr = mo;
  if (residual && (rc = make_tensor_map(ctx, &mr, dt, 2, residual, dout, sout, bout, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  GemmArgs g{bias, M, N, K, residual != nullptr, gamma};
  if (gamma) return launch_gemm<128, CB_EPI_NONE, true, true>(ctx, ma, mb, mo, mr, g, stream);
  return BN == 256 ? dispatch_gemm<256>(ctx, ma, mb, mo, mr, g, out_f32 != nullptr, epilogue, stream)
                   : dispatch_gemm<128>(ctx, ma, mb, mo, mr, g, out_f32 != nullptr, epilogue, stream);
}

int gemm_f16(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* residual, float* out_f32, void* out_f16, int M,
             int N, int K, int epilogue, cudaStream_t stream) {
  return gemm_f16_ex(ctx, A, W, bias, nullptr, residual, out_f32, out_f16, M, N, K, epilogue, stream);
}

}  // namespace cb

extern "C" int cb_gemm_f16_ex(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* gamma, const float* residual,
                              float* out_f32, void* out_f16, int M, int N, int K, int epilogue, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::gemm_f16_ex(ctx, A, W, bias, gamma, residual, out_f32, out_f16, M, N, K, epilogue, (cudaStream_t)stream);
}

extern "C" int cb_gemm_f16(cb_ctx* ctx, const void* A, const void* W, const float* bias, const float* residual, float* out_f32,
                           void* out_f16, int M, int N, int K, int epilogue, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::gemm_f16(ctx, A, W, bias, residual, out_f32, out_f16, M, N, K, epilogue, (cudaStream_t)stream);
}
