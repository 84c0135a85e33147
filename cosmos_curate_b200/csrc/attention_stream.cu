// softmax(Q K^T / sqrt(d)) V on the Hopper tensor cores (wgmma) for head_dim 88 and long sequences (InternVideo2-1B: T = 1025 at
// 4 frames, 2049 at 8), keys and values streamed.
//
// Unit of work: (clip, head, 128 query rows); persistent CTAs (one per SM) walk the units with the query block fastest, so the
// CTAs working on one (clip, head) at a time share its K and V in L2.
//
// Operand tiles come from a rank-5 TMA map over the packed QKV tensor, {88, heads, 3, T, n}: a box of 64 columns starting at
// column 64 reaches past 88 and TMA fills columns 88..127 with zeros (never the next head's columns, nor V's), and rows past the
// clip's own T are zero-filled too (never the next clip's tokens: an Inf or NaN there would turn 0 * V into NaN).  Each operand
// tile is two 128-byte-swizzled column atoms: columns 0..63 and 64..127.
//
// Warp roles (384 threads):
//   warpgroup 0, warp 0: TMA producer.  Q of a unit (128 rows, two atoms, 32 KB) into a two-deep Q buffer; K and V blocks of 128
//                keys (64 KB) into a two-deep ring.
//   warpgroups 1-2: query rows 64c..64c+63 of the unit.  Per key block: S = Q K^T (six k16 steps: columns 0..95, the last eight
//                zero) in registers, online softmax in fp32 (running max and row sum, accumulator rescaled per block), P packed to
//                fp16 in place as the register A operand of O += P V (V consumed from its [key][dim] rows as an MN-major B operand,
//                two n64 products for dims 0..63 and 64..127).  Keys past T are masked; query rows past T are not stored.
#include <cstdlib>

#include "common.h"
#include "ptx.cuh"

namespace cb {

constexpr int kAsThreads = 384;
constexpr int kAsHd = 88;
constexpr int kAsRows = 128;   // query rows per unit, and keys per streamed block
constexpr int kAsAtom = kAsRows * 128;  // one 64-column atom of a 128-row tile: 16 KB
constexpr int kAsQ = 0;                 // [2 buffers][2 atoms][128 rows][128 B]
constexpr int kAsKV = 4 * kAsAtom;      // [2 stages][K atom 0, K atom 1, V atom 0, V atom 1]
constexpr int kAsStage = 4 * kAsAtom;
constexpr int kAsBar = kAsKV + 2 * kAsStage;
constexpr int kAsSmem = kAsBar + 64 + 1024 /* alignment slack */;
static_assert(kAsSmem <= 232448, "shared memory budget");

struct AttnStreamArgs {
  __half* out;
  int tokens, heads, n_units, q_blocks;  // n_units = clips * heads * q_blocks
  float scale_log2e;
};

__device__ __forceinline__ float as_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t as_pack2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(kAsThreads, 1) attention_stream_kernel(const __grid_constant__ CUtensorMap map, const AttnStreamArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + kAsBar);
  uint64_t* q_empty = q_full + 2;
  uint64_t* kv_full = q_empty + 2;
  uint64_t* kv_empty = kv_full + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = a.tokens, k_blocks = (T + kAsRows - 1) / kAsRows;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&q_full[i], 1), mbar_init(&q_empty[i], 2);  // one arrival per consumer warpgroup
      mbar_init(&kv_full[i], 1), mbar_init(&kv_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dealloc<24>();
    if (warp == 0 && lane == 0) {  // ===== TMA producer
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;
      for (int u = blockIdx.x; u < a.n_units; u += gridDim.x, ++it) {
        const int qb = u % a.q_blocks, ch = u / a.q_blocks, clip = ch / a.heads, h = ch - clip * a.heads;
        const int qs = it & 1;
        uint8_t* sq = smem + kAsQ + qs * 2 * kAsAtom;
        mbar_wait_parked(&q_empty[qs], ((it >> 1) & 1) ^ 1);
        mbar_expect_tx(&q_full[qs], 2 * kAsAtom);
        for (int at = 0; at < 2; ++at) tma_load_5d(sq + at * kAsAtom, &map, &q_full[qs], 64 * at, h, 0, qb * kAsRows, clip);
        for (int kb = 0; kb < k_blocks; ++kb) {
          uint8_t* st = smem + kAsKV + stage * kAsStage;
          mbar_wait_parked(&kv_empty[stage], phase ^ 1);
          mbar_expect_tx(&kv_full[stage], kAsStage);
          for (int which = 1; which <= 2; ++which)  // K, then V
            for (int at = 0; at < 2; ++at)
              tma_load_5d(st + ((which - 1) * 2 + at) * kAsAtom, &map, &kv_full[stage], 64 * at, h, which, kb * kAsRows, clip);
          if (++stage == 2) stage = 0, phase ^= 1;
        }
      }
    }
  } else {  // ===== consumers: warpgroup c owns query rows 64c..64c+63 of the unit
    reg_alloc<240>();
    const int c = (warp >> 2) - 1, quad = lane & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const int r_in = (warp & 3) * 16 + (lane >> 2);  // this thread's first row inside the 64-row tile; the second is r_in + 8
    const int hidden = a.heads * kAsHd;
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int u = blockIdx.x; u < a.n_units; u += gridDim.x, ++it) {
      const int qb = u % a.q_blocks, ch = u / a.q_blocks, clip = ch / a.heads, h = ch - clip * a.heads;
      const int qs = it & 1;
      const uint32_t sq = smem_u32(smem + kAsQ + qs * 2 * kAsAtom + c * 64 * 128);
      mbar_wait_parked(&q_full[qs], (it >> 1) & 1);
      float o[64];  // o[0..31]: dims 0..63, o[32..63]: dims 64..127 (88.. are zero)
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = 0.f;
      float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll 1
      for (int kb = 0; kb < k_blocks; ++kb) {
        const uint32_t st = smem_u32(smem + kAsKV + stage * kAsStage);
        mbar_wait(&kv_full[stage], phase);
        float sc[64];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 6; ++k) {  // head dims 16k .. 16k + 15: atom k / 4, 32-byte step k % 4 inside it
          const uint32_t off = (uint32_t)((k >> 2) * kAsAtom);
          wgmma_m64n128k16(sc, wgmma_desc_sw128(sq + off) + (uint64_t)(2 * (k & 3)), wgmma_desc_sw128(st + off) + (uint64_t)(2 * (k & 3)), k != 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (kb == k_blocks - 1 && leader) mbar_arrive(&q_empty[qs]);  // Q is read by the QK^T products only
        // sc[4j + 2hh + e] = S(row r_in + 8hh, key kb*128 + 8j + 2quad + e)
        const int key0 = kb * kAsRows + 2 * quad;
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (key0 + 8 * j + (e & 1) >= T) sc[4 * j + e] = -INFINITY;
            mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * j + e]);
          }
        float mb[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
          mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
          const float corr = as_ex2((m[hh] - mx[hh]) * a.scale_log2e);  // exp2(-inf) = 0 on the first block
          m[hh] = mx[hh];
          l[hh] *= corr;
#pragma unroll
          for (int j = 0; j < 16; ++j) o[4 * j + 2 * hh] *= corr, o[4 * j + 2 * hh + 1] *= corr;
          mb[hh] = mx[hh] * a.scale_log2e;
        }
        uint32_t pa[32];  // pa[4ks .. 4ks + 3]: the A fragment of k-step ks (keys 16ks .. 16ks + 15 of the block)
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const float p0 = as_ex2(fmaf(sc[4 * j + 2 * hh], a.scale_log2e, -mb[hh]));
            const float p1 = as_ex2(fmaf(sc[4 * j + 2 * hh + 1], a.scale_log2e, -mb[hh]));
            l[hh] += p0 + p1;
            pa[2 * j + hh] = as_pack2(p0, p1);
          }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          wgmma_m64n64k16_ra_tb(o, pa + 4 * ks, wgmma_desc_sw128_mn(st + 2 * kAsAtom + ks * 2048), 1);
          wgmma_m64n64k16_ra_tb(o + 32, pa + 4 * ks, wgmma_desc_sw128_mn(st + 3 * kAsAtom + ks * 2048), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 32; ++i) asm volatile("" ::"r"(pa[i]));  // the A fragments stay in their registers until the MMAs have read them
        if (leader) mbar_arrive(&kv_empty[stage]);
        if (++stage == 2) stage = 0, phase ^= 1;
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
        const int row = qb * kAsRows + c * 64 + r_in + 8 * hh;
        if (row >= T) continue;
        const float inv = 1.0f / l[hh];
        __half* orow = a.out + ((size_t)clip * T + row) * hidden + h * kAsHd + 2 * quad;
#pragma unroll
        for (int j = 0; j < 11; ++j)  // dims 8j + 2quad + 0..1 < 88
          *reinterpret_cast<uint32_t*>(orow + 8 * j) = as_pack2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
      }
    }
  }
}

int attention_stream_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream) {
  if (head_dim != kAsHd) return fail(ctx, CB_ERR_UNSUPPORTED, "attention_stream: head_dim %d unsupported (88 only)", head_dim);
  if (!qkv || !out) return fail(ctx, CB_ERR_ARG, "attention_stream: null operand");
  if (n < 0 || tokens <= 0 || heads <= 0) return fail(ctx, CB_ERR_ARG, "attention_stream: bad shape n=%d tokens=%d heads=%d", n, tokens, heads);
  if (((uintptr_t)qkv & 15) || ((uintptr_t)out & 3)) return fail(ctx, CB_ERR_ARG, "attention_stream: qkv must be 16-byte, out 4-byte aligned");
  if (n == 0) return CB_OK;
  const uint64_t hidden = (uint64_t)heads * kAsHd;
  // {dim, head, q|k|v, token, clip}: boxes past column 88 and past the clip's T are zero-filled by TMA
  const uint64_t dims[5] = {(uint64_t)kAsHd, (uint64_t)heads, 3, (uint64_t)tokens, (uint64_t)n};
  const uint64_t strides[4] = {kAsHd * 2, hidden * 2, 3 * hidden * 2, (uint64_t)tokens * 3 * hidden * 2};
  const uint32_t box[5] = {64, 1, 1, kAsRows, 1};
  CUtensorMap map;
  int rc = make_tensor_map(ctx, &map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, qkv, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  static bool attr_done[64] = {};  // the attribute is per device: one process may drive several
  bool& attr_set = attr_done[ctx->device & 63];
  if (!attr_set) {
    CB_CUDA(ctx, cudaFuncSetAttribute(attention_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAsSmem));
    attr_set = true;
  }
  const int q_blocks = (tokens + kAsRows - 1) / kAsRows;
  const long long units = (long long)n * heads * q_blocks;
  if (units > 0x7fffffff) return fail(ctx, CB_ERR_UNSUPPORTED, "attention_stream: too many work units");
  AttnStreamArgs a{(__half*)out, tokens, heads, (int)units, q_blocks, 1.4426950408889634f / sqrtf((float)kAsHd)};
  const int grid = (int)std::min<long long>(units, ctx->sm_count);
  mark_launch(ctx, CB_PROF_ATTENTION, stream);
  attention_stream_kernel<<<grid, kAsThreads, kAsSmem, stream>>>(map, a);
  CB_CUDA(ctx, cudaGetLastError());
  return CB_OK;
}

}  // namespace cb

extern "C" int cb_attention_stream_f16(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, void* stream) {
  if (!ctx) return CB_ERR_ARG;
  return cb::attention_stream_f16(ctx, qkv, out, n, tokens, heads, head_dim, (cudaStream_t)stream);
}
