// wgmma attention for head_dim 128: the causal GQA prefill of the Qwen2.5-VL decoder (28 query / 4 K-V heads;
// call sites of the reference: internvla_n1.py L206 / L338 -> Qwen2_5_VLAttention with attn_implementation =
// "flash_attention_2", internvla_n1_policy.py L33-38).  Replaces the mma.sync kernel (attention.cu, attn_kernel<128>)
// for sequences of up to 320 keys, which covers the benchmark prompts (S = 304); longer sequences keep the old kernel.
//
// Work item = (sequence, K/V head).  K and V of the item (<= 320 rows x 128) are TMA-loaded ONCE into shared memory and
// serve the 7 query heads of the GQA group x ceil(S / 128) query tiles:
//
//   warp 8           TMA producer: K, V per item (128-byte swizzle, [rows][64] tiles), Q per query tile
//   warpgroups 0-1   64 query rows each, flash-attention style over 64-key blocks (causal blocks above the diagonal are
//                    never issued):  S = Q K^T  (wgmma m64n64k16, fp32 scores in registers) -> online softmax in registers
//                    (row max / sum across the 4 lanes that share a row) -> P packed to bf16 pairs IS the A-fragment
//                    layout, so  O += P V  takes P from registers (m64n128k16) and V in place as an MN-major B operand --
//                    no transpose, and neither scores nor probabilities touch shared memory.  One warpgroup's softmax runs
//                    under the other's MMAs.  Finally O / sum -> global.
#include <math.h>

#include <mutex>

#include "n1_ops.h"
#include "n1_ptx.cuh"

namespace n1 {
namespace {

constexpr int HD = 128, BQ = 128, BKEY = 64, KMAX = 320;
constexpr int kKBlock = KMAX * 128;             // bytes of one 64-column half of K (or V): 320 rows x 128 B = 40960
constexpr int kKVBytes = 2 * kKBlock;           // 81920
constexpr int kQBytes = BQ * HD * 2;            // 32768: two [128 x 64] k-blocks
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 32;  // 288
constexpr int kSmem = 2 * kKVBytes + kQBytes + 128 + 1024;
static_assert(kSmem <= 232448, "attention_wgmma: shared memory budget");

struct TcArgs {
  const int* cu_q;      // [batch + 1] token offsets (query == key sequences: self-attention prefill)
  int batch, heads_q, heads_kv;
  int causal;
  float scale_log2;     // softmax scale * log2(e)
  bf16* o;
  int ldo;
  int num_items;        // batch * heads_kv
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kThreads, 1)
attn_wgmma128_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const TcArgs args) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = sK + kKVBytes;
  uint8_t* sQ = sV + kKVBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sQ + kQBytes);
  uint64_t* kv_full = bars;       // K and V of the item landed
  uint64_t* kv_empty = bars + 1;  // every consumer warp is done with the item's K and V
  uint64_t* q_full = bars + 2;
  uint64_t* q_empty = bars + 3;   // every consumer warp's Q K^T MMAs of the tile are complete

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = args.heads_q / args.heads_kv;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ), tma_prefetch_desc(&tmK), tma_prefetch_desc(&tmV);
    mbar_init(kv_full, 1), mbar_init(kv_empty, kConsumerWarps), mbar_init(q_full, 1), mbar_init(q_empty, kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      uint32_t kv_ph = 0, q_ph = 0;
      for (int item = blockIdx.x; item < args.num_items; item += gridDim.x) {
        const int b = item / args.heads_kv, kh = item % args.heads_kv;
        const int start = args.cu_q[b], len = args.cu_q[b + 1] - start;
        mbar_wait(kv_empty, kv_ph ^ 1);
        kv_ph ^= 1;
        mbar_arrive_expect_tx(kv_full, 2 * kKVBytes);
        for (int kb = 0; kb < 2; ++kb)
          for (int r = 0; r < 2; ++r) {  // 320 rows as two boxes of 160 (rows past the sequence are masked / weigh 0)
            tma_load_2d(sK + kb * kKBlock + r * 160 * 128, &tmK, kv_full, kh * HD + kb * 64, start + r * 160);
            tma_load_2d(sV + kb * kKBlock + r * 160 * 128, &tmV, kv_full, kh * HD + kb * 64, start + r * 160);
          }
        const int q_tiles = (len + BQ - 1) / BQ;
        for (int hq = 0; hq < group; ++hq)
          for (int qt = 0; qt < q_tiles; ++qt) {
            mbar_wait(q_empty, q_ph ^ 1);
            q_ph ^= 1;
            mbar_arrive_expect_tx(q_full, kQBytes);
            for (int kb = 0; kb < 2; ++kb)
              tma_load_2d(sQ + kb * 16384, &tmQ, q_full, (kh * group + hq) * HD + kb * 64, start + qt * BQ);
          }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: 64 query rows per warpgroup
    const int wg = warp >> 2;
    const int quad = lane & 3;
    const int r_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows: r_in_tile and r_in_tile + 8
    uint32_t kv_ph = 0, q_ph = 0;
    for (int item = blockIdx.x; item < args.num_items; item += gridDim.x) {
      const int b = item / args.heads_kv, kh = item % args.heads_kv;
      const int start = args.cu_q[b], len = args.cu_q[b + 1] - start;
      const int q_tiles = (len + BQ - 1) / BQ;
      mbar_wait(kv_full, kv_ph);
      kv_ph ^= 1;
      for (int hq = 0; hq < group; ++hq)
        for (int qt = 0; qt < q_tiles; ++qt) {
          // keys this warpgroup's rows can see: causal -> up to the end of its own 64 rows
          const int k_hi = args.causal ? min(len, qt * BQ + wg * 64 + 64) : len;
          const int k_blocks = (k_hi + BKEY - 1) / BKEY;
          int vis[2];  // keys [0, vis) are visible to the row
#pragma unroll
          for (int h = 0; h < 2; ++h) vis[h] = args.causal ? min(len, qt * BQ + r_in_tile + h * 8 + 1) : len;
          float o[64];
#pragma unroll
          for (int i = 0; i < 64; ++i) o[i] = 0.f;
          float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
          mbar_wait(q_full, q_ph);
          q_ph ^= 1;
#pragma unroll 1
          for (int n = 0; n < k_blocks; ++n) {
            // ---- S = Q K^T for 64 keys: 2 k-blocks x 4 k-steps
            float s[32];
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
              const uint64_t ad = wgmma_desc_sw128(smem_u32(sQ + kb * 16384 + wg * 8192));
              const uint64_t bd = wgmma_desc_sw128(smem_u32(sK + kb * kKBlock + n * BKEY * 128));
#pragma unroll
              for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(s, ad + 2 * k, bd + 2 * k, (kb | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (n == k_blocks - 1) {  // the tile's last read of Q
              __syncwarp();
              if (lane == 0) mbar_arrive(q_empty);
            }
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
              alpha[h] = fast_exp2((mx[h] - m) * args.scale_log2);
              mx[h] = m;
              m_s[h] = m * args.scale_log2;
              sum[h] *= alpha[h];
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              o[4 * j + 0] *= alpha[0], o[4 * j + 1] *= alpha[0];
              o[4 * j + 2] *= alpha[1], o[4 * j + 3] *= alpha[1];
            }
            // ---- P -> bf16 A fragments (k-step ks = keys 16 ks .. 16 ks + 15 of the block) and O += P V
            uint32_t pa[4][4];
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int kk = k0 + j * 8;
                const float p0 = kk < vis[h] ? fast_exp2(s[4 * j + 2 * h] * args.scale_log2 - m_s[h]) : 0.f;
                const float p1 = kk + 1 < vis[h] ? fast_exp2(s[4 * j + 2 * h + 1] * args.scale_log2 - m_s[h]) : 0.f;
                sum[h] += p0 + p1;
                pa[j >> 1][(j & 1) * 2 + h] = pack_bf16(p0, p1);
              }
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
              // V as stored ([keys][64 head-dim values] rows of 128 bytes): 8 keys form a 1024-byte atom (SBO), the second
              // 64-wide half of the head dimension lies kKBlock bytes further (LBO)
              const uint64_t bd = wgmma_desc_sw128(smem_u32(sV + (n * BKEY + ks * 16) * 128), kKBlock);
              wgmma_rs<1>(o, pa[ks], bd, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
          }
          // ---- epilogue: O / sum -> global
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float l = sum[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = l > 0.f ? 1.0f / l : 0.f;
            const int q_pos = qt * BQ + r_in_tile + h * 8;
            if (q_pos < len) {
              bf16* orow = args.o + (long)(start + q_pos) * args.ldo + (kh * group + hq) * HD + quad * 2;
#pragma unroll
              for (int j = 0; j < 16; ++j)
                *reinterpret_cast<uint32_t*>(orow + j * 8) = pack_bf16(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
            }
          }
        }
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty);
    }
  }
}

}  // namespace

bool attention_tc_supported(const AttnParams& p) {
  return p.hd == HD && p.cu_q != nullptr && p.cu_k == p.cu_q && !p.k_len && p.kv_div == 1 && p.max_seq_q > 0 &&
         p.max_seq_q <= KMAX && p.total_rows > 0 && p.heads_q % p.heads_kv == 0 && p.ldq % 8 == 0 && p.ldk % 8 == 0 &&
         p.ldv % 8 == 0 && p.ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(p.q) & 15) == 0 &&
         (reinterpret_cast<uintptr_t>(p.k) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.v) & 15) == 0 &&
         (reinterpret_cast<uintptr_t>(p.o) & 15) == 0;
}

void attention_tc128(const AttnParams& p, cudaStream_t stream) {
  N1_CHECK(attention_tc_supported(p), "attention_tc128: unsupported arguments");
  static std::once_flag once;
  std::call_once(once, [] { cudaFuncSetAttribute(attn_wgmma128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem); });
  const long rows = p.total_rows;
  CUtensorMap tmQ = tma_map_2d(p.q, rows, (long)p.heads_q * HD, p.ldq, BQ, 64, true);
  CUtensorMap tmK = tma_map_2d(p.k, rows, (long)p.heads_kv * HD, p.ldk, 160, 64, true);
  CUtensorMap tmV = tma_map_2d(p.v, rows, (long)p.heads_kv * HD, p.ldv, 160, 64, true);
  TcArgs a;
  a.cu_q = p.cu_q, a.batch = p.batch, a.heads_q = p.heads_q, a.heads_kv = p.heads_kv, a.causal = p.causal;
  a.scale_log2 = p.scale * 1.4426950408889634f;
  a.o = p.o, a.ldo = p.ldo, a.num_items = p.batch * p.heads_kv;
  const int grid = a.num_items < device_sm_count() ? a.num_items : device_sm_count();
  attn_wgmma128_kernel<<<grid, kThreads, kSmem, stream>>>(tmQ, tmK, tmV, a);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

}  // namespace n1
