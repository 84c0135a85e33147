// softmax(Q K^T / sqrt(d)) V on the Hopper tensor cores (wgmma) for the ViT-L/14 shape class: head_dim 64, 129..257 tokens.
//
// 257 = 4 * 64 + 1: the first 256 tokens map onto the tensor cores with no padding at all - four 64-row query tiles against
// one 256-key tile (S = Q K^T is one chain of wgmma m64n256k16 per query tile; no online softmax, every key of the row is in
// the warpgroup's registers at once).  Token 256 rides along as a ninth..sixteenth of a tile: its key is one more N = 8 product
// (columns past the first masked), its value one more k-step of P V, and its query row is computed on SIMT by three warps.
// Persistent CTAs (one per SM) loop over (image, head) units; Q, K and V of a unit arrive by TMA into a two-deep ring.
//
// Warp roles (384 threads):
//   warpgroup 0  warp 0: TMA producer (Q 32 + 1 KB, K 32 + 1 KB, V 32 + 2 KB per unit from the [n][T][3*hidden] QKV tensor)
//                warps 1-3: query row 256 on SIMT from smem Q/K/V: each warp takes a third of the 257 dot products of 64,
//                every warp forms the softmax, each takes a third of the keys of the weighted sum, warp 1 adds the thirds
//   warpgroups 1-2  query rows 0..127 / 128..255, 64 at a time, taking turns on the tensor cores: S in registers (128 per
//                thread), row max / exp2 / row sum with quad shuffles, P packed to fp16 IN PLACE as the register A operand of O = P V (the accumulator layout of S is
//                the A layout of the next product; V is consumed straight from its [key][dim] rows as an MN-major B operand,
//                no transpose pass), O / rowsum -> fp16 -> global.
#include <cstdlib>
#include <cstring>

#include "common.h"
#include "ptx.cuh"

namespace cb {

constexpr int kAtThreads = 384;
constexpr int kAtQ = 0;                       // 256 rows x 128 B, SW128
constexpr int kAtK = 32768;                   // 256 rows, then the 8-row tile that starts at token 256
constexpr int kAtV = kAtK + 32768 + 1024;     // 256 rows, then the 16-row tile that starts at token 256
constexpr int kAtQx = kAtV + 32768 + 2048;    // the 8-row Q tile that starts at token 256
constexpr int kAtStage = kAtQx + 1024;        // 102400 B: a multiple of 1024
constexpr int kAtPx = 2 * kAtStage;           // query row 256: [260] fp32 scores, [256] probabilities, [3][64] partial outputs
constexpr int kAtBar = kAtPx + 3072;
constexpr int kAtSmem = kAtBar + 64 + 1024 /* alignment slack */;
static_assert(kAtStage % 1024 == 0 && kAtSmem <= 232448, "shared memory budget");

struct AttnArgs {
  const __half* qkv;
  __half* out;
  int tokens, heads, n_units;  // n_units = images * heads
  float scale_log2e;
};

// named barriers: 1 = the three row-256 warps; 2 + c = consumer warpgroup c may issue its next product
constexpr int kAtBarRow256 = 1, kAtBarIssue = 2;

__device__ __forceinline__ void named_bar_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// FULL: tokens is 256 or 257, i.e. every column / row of the tensor-core tiles is a real token (no masking code at all)
template <bool FULL>
__global__ void __launch_bounds__(kAtThreads, 1) attention_wgmma_kernel(const __grid_constant__ CUtensorMap map_qkv, const __grid_constant__ CUtensorMap map_k8,
                                                                         const __grid_constant__ CUtensorMap map_v16, const AttnArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - smem_u32(smem_raw));
  float* px = reinterpret_cast<float*>(smem + kAtPx);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kAtBar);
  uint64_t* empty = full + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = a.tokens, hidden = a.heads * 64;
  const bool has_extra = T == 257;
  const int t_mma = FULL ? 256 : (T < 256 ? T : 256);  // keys / query rows living in the tensor-core tiles

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_qkv);
    for (int i = 0; i < 2; ++i) mbar_init(&full[i], 1), mbar_init(&empty[i], 9);  // 8 consumer warps + the row-256 warp
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dealloc<72>();  // 72 x 128 + 216 x 256 = 168 x 384, the registers the CTA was launched with
    if (warp == 0) {
      if (lane == 0) {  // ===== TMA producer
        int it = 0;
        for (int u = blockIdx.x; u < a.n_units; u += gridDim.x, ++it) {
          const int img = u / a.heads, h = u - img * a.heads, s = it & 1;
          uint8_t* st = smem + s * kAtStage;
          mbar_wait_parked(&empty[s], ((it >> 1) & 1) ^ 1);
          mbar_expect_tx(&full[s], 3 * 32768 + (has_extra ? 1024 + 2048 + 1024 : 0));
          for (int half = 0; half < 2; ++half) {
            tma_load_3d(st + kAtK + half * 16384, &map_qkv, &full[s], hidden + h * 64, half * 128, img);
            tma_load_3d(st + kAtQ + half * 16384, &map_qkv, &full[s], h * 64, half * 128, img);
          }
          if (has_extra) {
            tma_load_3d(st + kAtK + 32768, &map_k8, &full[s], hidden + h * 64, 256, img);
            tma_load_3d(st + kAtQx, &map_k8, &full[s], h * 64, 256, img);
          }
          for (int half = 0; half < 2; ++half) tma_load_3d(st + kAtV + half * 16384, &map_qkv, &full[s], 2 * hidden + h * 64, half * 128, img);
          if (has_extra) tma_load_3d(st + kAtV + 32768, &map_v16, &full[s], 2 * hidden + h * 64, 256, img);
        }
      }
    } else {  // ===== query row 256 on SIMT, warps 1-3 (96 threads)
      const int t96 = threadIdx.x - 32, w3 = t96 >> 5;
      float* sc_x = px;            // [257] scores of query row 256
      float* p_x256 = px + 260;    // [256] its probabilities
      float* o_part = px + 516;    // [3][64] per-warp partial P.V
      int it = 0;
      for (int u = blockIdx.x; u < a.n_units; u += gridDim.x, ++it) {
        const int img = u / a.heads, h = u - img * a.heads, s = it & 1;
        const size_t row0 = (size_t)img * T;
        const uint8_t* sK = smem + s * kAtStage + kAtK;
        const uint8_t* sV = smem + s * kAtStage + kAtV;
        const uint8_t* sQx = smem + s * kAtStage + kAtQx;  // query row 256 is row 0 of its tile: unswizzled
        mbar_wait_parked(&full[s], (it >> 1) & 1);
        if (has_extra) {
          // scores: thread t96 owns keys t96, t96 + 96, t96 + 192 (< 257; key 256 is row 0 of the 8-row tile right after key 255,
          // so the 128-byte swizzle formula holds for it too).  Each dot runs in the same order as a plain 64-term fma chain.
          float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const uint4 qj = *reinterpret_cast<const uint4*>(sQx + (j << 4));
            const __half2* q2 = reinterpret_cast<const __half2*>(&qj);
#pragma unroll
            for (int i = 0; i < 3; ++i) {
              const int key = t96 + 96 * i;
              if (key > 256) continue;
              const uint4 kb = *reinterpret_cast<const uint4*>(sK + key * 128 + ((j ^ (key & 7)) << 4));
              const __half2* k2 = reinterpret_cast<const __half2*>(&kb);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 qf = __half22float2(q2[e]), kf = __half22float2(k2[e]);
                acc[i] = fmaf(qf.x, kf.x, acc[i]), acc[i] = fmaf(qf.y, kf.y, acc[i]);
              }
            }
          }
#pragma unroll
          for (int i = 0; i < 3; ++i)
            if (t96 + 96 * i <= 256) sc_x[t96 + 96 * i] = acc[i];
          named_bar_sync(kAtBarRow256, 96);
          // softmax, computed redundantly by each warp (lane owns keys lane + 32 i): every warp holds the row max and sum, and writes
          // the probabilities of its own P.V key range [lo, hi) - ranges are multiples of 4 for the float4 reads below
          const int lo = w3 == 0 ? 0 : (w3 == 1 ? 88 : 172), hi = w3 == 0 ? 88 : (w3 == 1 ? 172 : 256);
          float sc[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) sc[i] = sc_x[lane + 32 * i];
          const float s_x = sc_x[256];
          float mx = s_x;
#pragma unroll
          for (int i = 0; i < 8; ++i) mx = fmaxf(mx, sc[i]);
          for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
          const float mb = mx * a.scale_log2e;
          float sum = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int key = lane + 32 * i;
            const float p = ex2f(fmaf(sc[i], a.scale_log2e, -mb));
            if (key >= lo && key < hi) p_x256[key] = p;
            sum += p;
          }
          for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
          const float p_x = ex2f(fmaf(s_x, a.scale_log2e, -mb));
          sum += p_x;
          __syncwarp();
          // P.V over this warp's keys: lane owns output dims 2*lane, 2*lane+1 = byte lane*4 of every V row -> 16-byte chunk lane>>2
          const uint8_t* vbase = sV + (lane & 3) * 4;
          const int ch = lane >> 2;
          float oa[4] = {0.f, 0.f, 0.f, 0.f}, ob[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
          for (int key = lo; key < hi; key += 4) {
            const float4 p4 = *reinterpret_cast<const float4*>(p_x256 + key);
            const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {  // four independent accumulator pairs: the loop is not an FMA latency chain
              const int kk = key + e;
              const float2 vf = __half22float2(*reinterpret_cast<const __half2*>(vbase + kk * 128 + ((ch ^ (kk & 7)) << 4)));
              oa[e] = fmaf(pv[e], vf.x, oa[e]), ob[e] = fmaf(pv[e], vf.y, ob[e]);
            }
          }
          *reinterpret_cast<float2*>(o_part + w3 * 64 + 2 * lane) = make_float2((oa[0] + oa[1]) + (oa[2] + oa[3]), (ob[0] + ob[1]) + (ob[2] + ob[3]));
          named_bar_sync(kAtBarRow256, 96);
          if (w3 == 0) {
            const float2 o0 = *reinterpret_cast<const float2*>(o_part + 2 * lane), o1 = *reinterpret_cast<const float2*>(o_part + 64 + 2 * lane),
                         o2 = *reinterpret_cast<const float2*>(o_part + 128 + 2 * lane);
            float ox = (o0.x + o1.x) + o2.x, oy = (o0.y + o1.y) + o2.y;
            const float2 vxf = __half22float2(*reinterpret_cast<const __half2*>(sV + 32768 + lane * 4));  // row 0 of the tile: unswizzled
            ox = fmaf(p_x, vxf.x, ox), oy = fmaf(p_x, vxf.y, oy);
            const float inv = 1.0f / sum;
            *reinterpret_cast<uint32_t*>(a.out + (row0 + 256) * hidden + h * 64 + 2 * lane) = pack2(ox * inv, oy * inv);
          }
        }
        // warps 2 and 3 are past their last read of this stage (the barrier above); warp 1 releases it once for all three
        if (w3 == 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[s]);
        }
      }
    }
  } else {  // ===== consumers: warpgroup c owns query rows 128c..128c+127, 64 at a time
    reg_alloc<216>();
    const int c = (warp >> 2) - 1, quad = lane & 3;
    const int r_in = (warp & 3) * 16 + (lane >> 2);  // this thread's first row inside a 64-row tile; the second is r_in + 8
    // Ping-pong: the two warpgroups take turns to issue their products (S, P.V, S, P.V, ... each), so one warpgroup's
    // exp2 / sum runs while the other's product is on the tensor cores.  Warpgroup 0 goes first.
    const int my_turn = kAtBarIssue + c, their_turn = kAtBarIssue + 1 - c;
    if (c == 1) named_bar_arrive(their_turn, 256);
    int it = 0;
    for (int u = blockIdx.x; u < a.n_units; u += gridDim.x, ++it) {
      const int img = u / a.heads, h = u - img * a.heads, s = it & 1;
      const size_t row0 = (size_t)img * T;
      const uint32_t st = smem_u32(smem + s * kAtStage);
      mbar_wait_parked(&full[s], (it >> 1) & 1);
#pragma unroll 1
      for (int qt = 0; qt < 2; ++qt) {
        const int tile_row = c * 128 + qt * 64;
        if (!FULL && tile_row >= t_mma) {  // warpgroup-uniform: pass both turns of the skipped tile on
          for (int k = 0; k < 2; ++k) named_bar_sync(my_turn, 256), named_bar_arrive(their_turn, 256);
          continue;
        }
        const uint64_t dq = wgmma_desc_sw128(st + kAtQ + tile_row * 128), dk = wgmma_desc_sw128(st + kAtK);
        float sc[128], sx[4];
        named_bar_sync(my_turn, 256);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n256k16(sc, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k != 0);
        if (has_extra) {
          const uint64_t dkx = wgmma_desc_sw128(st + kAtK + 32768);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n8k16(sx, dq + (uint64_t)(2 * k), dkx + (uint64_t)(2 * k), k != 0);
        }
        wgmma_commit();
        named_bar_arrive(their_turn, 256);
        wgmma_wait<0>();
        // sc[4j + 2h + e] = S(row r_in + 8h, key 8j + 2 quad + e); key 256 of row r_in + 8h is sx[2h] of the quad's first lane
        const bool own_x = has_extra && quad == 0;
        float mx[2] = {own_x ? sx[0] : -INFINITY, own_x ? sx[2] : -INFINITY};
#pragma unroll
        for (int j = 0; j < 32; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (!FULL && 8 * j + 2 * quad + (e & 1) >= t_mma) sc[4 * j + e] = -INFINITY;
            mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * j + e]);
          }
        float mb[2], sum[2], p_x[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
          mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
          mb[hh] = mx[hh] * a.scale_log2e;
          p_x[hh] = own_x ? ex2f(fmaf(sx[2 * hh], a.scale_log2e, -mb[hh])) : 0.f;
          sum[hh] = p_x[hh];
        }
        // P = exp2(S * scale - max) -> fp16 pairs: pa[4ks .. 4ks + 3] is the A fragment of k-step ks (keys 16ks .. 16ks + 15)
        uint32_t pa[64];
#pragma unroll
        for (int j = 0; j < 32; ++j)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const float p0 = ex2f(fmaf(sc[4 * j + 2 * hh], a.scale_log2e, -mb[hh])), p1 = ex2f(fmaf(sc[4 * j + 2 * hh + 1], a.scale_log2e, -mb[hh]));
            sum[hh] += p0 + p1;
            pa[2 * j + hh] = pack2(p0, p1);
          }
        const uint32_t pax[4] = {pack2(p_x[0], 0.f), pack2(p_x[1], 0.f), 0u, 0u};  // key 256, then fifteen zero columns
        float o[32];
        named_bar_sync(my_turn, 256);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 16; ++ks) wgmma_m64n64k16_ra_tb(o, pa + 4 * ks, wgmma_desc_sw128_mn(st + kAtV + ks * 2048), ks != 0);
        if (has_extra) wgmma_m64n64k16_ra_tb(o, pax, wgmma_desc_sw128_mn(st + kAtV + 32768), 1);
        wgmma_commit();
        named_bar_arrive(their_turn, 256);
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 64; ++i) asm volatile("" ::"r"(pa[i]));  // the A fragments stay in their registers until the MMAs have read them
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          sum[hh] += __shfl_xor_sync(0xffffffffu, sum[hh], 1);
          sum[hh] += __shfl_xor_sync(0xffffffffu, sum[hh], 2);
          const int row = tile_row + r_in + 8 * hh;
          if (!FULL && row >= t_mma) continue;
          const float inv = 1.0f / sum[hh];
          __half* orow = a.out + (row0 + row) * hidden + h * 64 + 2 * quad;
#pragma unroll
          for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(orow + 8 * j) = pack2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
  }
}

// host side: launches and sets *launched for the shape class this kernel serves; other shapes go to the mma.sync kernel
int attention_wgmma(cb_ctx* ctx, const void* qkv, void* out, int n, int tokens, int heads, int head_dim, cudaStream_t stream, bool* launched) {
  *launched = false;
  const char* sel = std::getenv("CB_ATTN_KERNEL");
  if (sel && std::strcmp(sel, "mma") == 0) return CB_OK;
  if (head_dim != 64 || tokens < 129 || tokens > 257) return CB_OK;
  const int hidden = heads * 64;
  CUtensorMap map, map_k8, map_v16;
  // rank 3, {3*hidden, T, n}: a tile never reaches into the next image.  TMA zero-fills its rows past the image's own T, so the
  // masked keys and query rows of a short image, and the rows past token 256 of the tiles below, hold zeros: P.V multiplies their
  // zero probabilities by 0, never by a neighbouring image's V (an Inf or NaN there would turn 0 * V into NaN).
  const uint64_t dims[3] = {(uint64_t)3 * hidden, (uint64_t)tokens, (uint64_t)n};
  const uint64_t strides[2] = {(uint64_t)3 * hidden * 2, (uint64_t)tokens * 3 * hidden * 2};
  const uint32_t box[3] = {64, 128, 1}, box8[3] = {64, 8, 1}, box16[3] = {64, 16, 1};
  int rc = make_tensor_map(ctx, &map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, qkv, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  // the tiles that start at token 256: one MMA n-step of keys, one MMA k-step of values.  Only their first row is a token (256);
  // the kernel gives the zero-filled rest zero probability.
  rc = make_tensor_map(ctx, &map_k8, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, qkv, dims, strides, box8, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  rc = make_tensor_map(ctx, &map_v16, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, qkv, dims, strides, box16, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  static bool attr_done[64] = {};  // the attribute is per device: one process may drive several
  bool& attr_set = attr_done[ctx->device & 63];
  if (!attr_set) {
    CB_CUDA(ctx, cudaFuncSetAttribute(attention_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAtSmem));
    CB_CUDA(ctx, cudaFuncSetAttribute(attention_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAtSmem));
    attr_set = true;
  }
  AttnArgs a{(const __half*)qkv, (__half*)out, tokens, heads, n * heads, 1.4426950408889634f / sqrtf(64.f)};
  const int grid = std::min(n * heads, ctx->sm_count);
  mark_launch(ctx, CB_PROF_ATTENTION, stream);
  if (tokens >= 256)
    attention_wgmma_kernel<true><<<grid, kAtThreads, kAtSmem, stream>>>(map, map_k8, map_v16, a);
  else
    attention_wgmma_kernel<false><<<grid, kAtThreads, kAtSmem, stream>>>(map, map_k8, map_v16, a);
  CB_CUDA(ctx, cudaGetLastError());
  *launched = true;
  return CB_OK;
}

}  // namespace cb
