// wgmma chunk attention over a slotted K/V cache, head_dim 128: the continuation prefill of a System-2 conversation,
// where a chunk of new query rows per sequence attends to every cached key of its slot (28 query / 4 K-V heads).
//
// Work item = (query tile, K/V head, sequence).  The G = heads_q / heads_kv query heads of a K/V head are folded into
// the M dimension: warpgroup w holds R = 64 / G query rows x G heads (row m = r * G + g; one 3-D TMA box of the packed
// q rows), so every K/V block is loaded once per GQA group instead of once per query head.
//
//   warp 8           producer: Q of the tile (TMA), then K / V in 64-key blocks through a kStages ring (TMA for whole
//                    blocks; the last, partial block of a sequence is copied by the warp with plain loads and its rows
//                    past the sequence zeroed, so no row past ctx + n of a slot is ever read).  On a paged pool a
//                    block is one page: its first row comes from the page table
//   warpgroups 0-1   S = Q K^T (wgmma m64n64k16) -> online softmax in registers -> O += P V (m64n128k16, P from
//                    registers, V in place as an MN-major B operand), as attention_wgmma.cu.  O / sum -> global.
#include <math.h>

#include <mutex>

#include "dec_tile.cuh"

namespace n1 {
namespace {

constexpr int HD = 128, BKEY = 64, kStages = 4;
constexpr int kHalf = BKEY * 128;                   // one 64-column half of a K (or V) block: 8192 bytes
constexpr int kBlockBytes = 2 * kHalf;              // 16384
constexpr int kStageBytes = 2 * kBlockBytes;        // K and V
constexpr int kQBytes = 2 * 128 * 128;              // two k-blocks of 128 folded rows
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 32;  // 288
constexpr int kSmem = kStages * kStageBytes + kQBytes + 256 + 1024;
static_assert(kSmem <= 232448, "attention_cache: shared memory budget");

struct CacheArgs {
  const bf16 *k, *v;
  int ldkv;
  bf16* o;
  int ldo;
  const int *cu_q, *ctx, *row0, *pages;
  int group, rows_wg;  // G query heads per K/V head, R = 64 / G query rows per warpgroup
  float scale_log2;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kThreads, 1)
attn_cache_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmV, const CacheArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + kQBytes;  // stage s: K at s * kStageBytes, V kBlockBytes further
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + kStages * kStageBytes);
  uint64_t* q_full = bars;
  uint64_t* full = bars + 1;
  uint64_t* empty = bars + 1 + kStages;

  const int b = blockIdx.z, kh = blockIdx.y;
  const int q_start = a.cu_q[b], n_q = a.cu_q[b + 1] - q_start;
  const int G = a.group, R = a.rows_wg;
  const int r0 = blockIdx.x * 2 * R;  // first query row of the tile within the chunk
  if (r0 >= n_q) return;
  const int ctx = a.ctx[b], k_len = ctx + n_q, row0 = a.row0[b];
  const int k_hi = min(k_len, ctx + r0 + 2 * R);  // keys any row of the tile can see
  const int n_blocks = (k_hi + BKEY - 1) / BKEY;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // rows 63 (G = 7) of each warpgroup's Q half are never written by the TMA: zero them so every score stays finite
  for (int i = threadIdx.x; i < kQBytes / 16; i += kThreads) reinterpret_cast<uint4*>(sQ)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ), tma_prefetch_desc(&tmK), tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < kStages; ++s) mbar_init(full + s, 1), mbar_init(empty + s, kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ------------------------------------------------------------------ producer warp
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, 4 * 128 * G * R);
      for (int wg = 0; wg < 2; ++wg)
        for (int kb = 0; kb < 2; ++kb)
          tma_load_3d(sQ + kb * 16384 + wg * 8192, &tmQ, q_full, kb * 64, kh * G, q_start + r0 + wg * R);
    }
    for (int n = 0; n < n_blocks; ++n) {
      const int st = n % kStages;
      mbar_wait(empty + st, ((n / kStages) & 1) ^ 1);
      uint8_t* sK = sKV + st * kStageBytes;
      uint8_t* sV = sK + kBlockBytes;
      const int key0 = n * BKEY, rem = k_len - key0;
      const int krow = a.pages ? a.pages[(row0 >> 6) + n] * BKEY : row0 + key0;  // first cache row of the block
      if (rem >= BKEY) {
        if (lane == 0) {
          mbar_arrive_expect_tx(full + st, kStageBytes);
          for (int kb = 0; kb < 2; ++kb) {
            tma_load_2d(sK + kb * kHalf, &tmK, full + st, kh * HD + kb * 64, krow);
            tma_load_2d(sV + kb * kHalf, &tmV, full + st, kh * HD + kb * 64, krow);
          }
        }
      } else {
        // partial last block: rows [0, rem) from global, the rest zero (P is 0 there, and 0 * V must stay 0)
        for (int i = lane; i < BKEY * 16; i += 32) {
          const int r = i >> 4, c = i & 15;
          uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
          if (r < rem) {
            const long g = (long)(krow + r) * a.ldkv + kh * HD + c * 8;
            kv = *reinterpret_cast<const uint4*>(a.k + g);
            vv = *reinterpret_cast<const uint4*>(a.v + g);
          }
          const int off = sw128_offset(r, c * 8);
          *reinterpret_cast<uint4*>(sK + off) = kv;
          *reinterpret_cast<uint4*>(sV + off) = vv;
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(full + st);
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: 64 folded rows per warpgroup
    const int wg = warp >> 2, quad = lane & 3;
    const int m_a = (warp & 3) * 16 + (lane >> 2);  // this thread's folded rows: m_a and m_a + 8
    int vis[2], qrow[2];                              // keys [0, vis) visible; query row within the chunk (-1: none)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m_a + h * 8;
      const int r = r0 + wg * R + m / G;
      qrow[h] = (m < G * R && r < n_q) ? r : -1;
      vis[h] = min(k_len, ctx + r + 1);
    }
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
    mbar_wait(q_full, 0);
#pragma unroll 1
    for (int n = 0; n < n_blocks; ++n) {
      const int st = n % kStages;
      const uint8_t* sK = sKV + st * kStageBytes;
      const uint8_t* sV = sK + kBlockBytes;
      mbar_wait(full + st, (n / kStages) & 1);
      float s[32];
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        const uint64_t ad = wgmma_desc_sw128(smem_u32(sQ + kb * 16384 + wg * 8192));
        const uint64_t bd = wgmma_desc_sw128(smem_u32(sK + kb * kHalf));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(s, ad + 2 * k, bd + 2 * k, (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // ---- online softmax: s[4 j + 2 h + e] = row h, key n * 64 + 8 j + 2 quad + e
      const int k0 = n * BKEY + quad * 2;
      float alpha[2], m_s[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float m = mx[h];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (k0 + j * 8 + e < vis[h]) m = fmaxf(m, s[4 * j + 2 * h + e]);
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        // key 0 is visible to every row, so m is finite from the first block on
        alpha[h] = fast_exp2((mx[h] - m) * a.scale_log2);
        mx[h] = m;
        m_s[h] = m * a.scale_log2;
        sum[h] *= alpha[h];
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        o[4 * j + 0] *= alpha[0], o[4 * j + 1] *= alpha[0];
        o[4 * j + 2] *= alpha[1], o[4 * j + 3] *= alpha[1];
      }
      uint32_t pa[4][4];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int kk = k0 + j * 8;
          const float p0 = kk < vis[h] ? fast_exp2(s[4 * j + 2 * h] * a.scale_log2 - m_s[h]) : 0.f;
          const float p1 = kk + 1 < vis[h] ? fast_exp2(s[4 * j + 2 * h + 1] * a.scale_log2 - m_s[h]) : 0.f;
          sum[h] += p0 + p1;
          pa[j >> 1][(j & 1) * 2 + h] = pack_bf16(p0, p1);
        }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        // V as stored ([keys][64 head-dim values], 128-byte rows): 8 keys form a 1024-byte atom (SBO), the second
        // 64-wide half of the head dimension lies kHalf bytes further (LBO)
        const uint64_t bd = wgmma_desc_sw128(smem_u32(sV + ks * 16 * 128), kHalf);
        wgmma_rs<1>(o, pa[ks], bd, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty + st);
    }
    // ---- epilogue: O / sum -> global
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = sum[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = l > 0.f ? 1.0f / l : 0.f;
      if (qrow[h] >= 0) {
        const int m = m_a + h * 8;
        bf16* orow = a.o + (long)(q_start + qrow[h]) * a.ldo + (kh * G + m % G) * HD + quad * 2;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          *reinterpret_cast<uint32_t*>(orow + j * 8) = pack_bf16(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
      }
    }
  }
}

}  // namespace

void attention_cache(const CacheAttnParams& p, cudaStream_t stream) {
  if (p.batch <= 0) return;
  N1_CHECK(p.heads_kv > 0 && p.heads_q % p.heads_kv == 0 && p.heads_q / p.heads_kv <= 64,
           "attention_cache: heads_q must be a multiple of heads_kv (at most 64 per group)");
  N1_CHECK(p.ldq % 8 == 0 && p.ldkv % 8 == 0 && p.ldo % 8 == 0 && p.max_chunk > 0 && p.q_rows > 0 && p.kv_rows > 0,
           "attention_cache: bad strides / sizes");
  N1_CHECK((reinterpret_cast<uintptr_t>(p.k) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.v) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(p.o) & 15) == 0,
           "attention_cache: 16-byte alignment");
  N1_CHECK(p.batch <= 65535 && p.heads_kv <= 65535, "attention_cache: grid too large");
  static std::once_flag once;
  std::call_once(once, [] { cudaFuncSetAttribute(attn_cache_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem); });
  CacheArgs a;
  a.k = p.k, a.v = p.v, a.ldkv = p.ldkv, a.o = p.o, a.ldo = p.ldo;
  a.cu_q = p.cu_q, a.ctx = p.ctx, a.row0 = p.row0, a.pages = p.pages;
  a.group = p.heads_q / p.heads_kv;
  a.rows_wg = 64 / a.group;
  a.scale_log2 = p.scale * 1.4426950408889634f;
  // q viewed as [rows][heads_q][128]: one box = R rows x the G heads of a group x 64 columns = R * G swizzled 128-byte rows
  const long qd[3] = {HD, p.heads_q, p.q_rows}, qs[2] = {HD, p.ldq};
  const int qb[3] = {64, a.group, a.rows_wg};
  CUtensorMap tmQ = tma_map_3d_sw128(p.q, qd, qs, qb);
  CUtensorMap tmK = tma_map_2d(p.k, p.kv_rows, (long)p.heads_kv * HD, p.ldkv, BKEY, 64, true);
  CUtensorMap tmV = tma_map_2d(p.v, p.kv_rows, (long)p.heads_kv * HD, p.ldkv, BKEY, 64, true);
  const int tiles = (p.max_chunk + 2 * a.rows_wg - 1) / (2 * a.rows_wg);
  dim3 grid(tiles, p.heads_kv, p.batch);
  attn_cache_kernel<<<grid, kThreads, kSmem, stream>>>(tmQ, tmK, tmV, a);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

}  // namespace n1
