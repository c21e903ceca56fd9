// Weight gradients without operand transposes:   dW[No, Ko] (+)= dY[M, No]^T · X[M, Ko]      (bf16 in, fp32 out)
//
// The contraction runs over the ROWS of both operands (M = tokens: 6 144 ... 98 304 in the System-1 training step), while
// the output is a small weight-shaped matrix (No, Ko <= a few thousand).  Transposing dY and X with a kernel to feed the
// K-major GEMM costs hundreds of launches per step, and one CTA per output tile leaves most SMs idle.  Here:
//   * both operands are read in place as MN-major wgmma operands: a TMA box of [64 rows x 64 columns] of the row-major
//     matrix (128-byte rows, 128-byte swizzle) IS the canonical MN-major layout -- 8 rows form a 1024-byte atom (SBO), the
//     second 64-wide half of the 128-wide tile lies one box (8 KB, LBO) further; a k-step of 16 rows advances 2 KB
//     (same layout as V in attention_wgmma.cu; here both the A and the B operand are transposed by the instruction);
//   * the M range is SPLIT over CTAs (grid = output tiles x splits ~ SM count); partial tiles go to an fp32
//     workspace and a second kernel sums them in a fixed order into the target (deterministic; `accumulate` adds onto
//     the gradient already in the bucket).
// Reference: autograd of every nn.Linear of the trainable System-1 branches (navdp.py L291-312 loss.backward()).
// Tensor bound: 2 · M · No · Ko flop; HBM traffic = both operands once per output-tile column / row they belong to.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "bwd_kernels.h"
#include "n1_ops.h"
#include "n1_ptx.cuh"

namespace n1 {
namespace {

constexpr int BM = 128, BN = 128, KB = 64;           // output tile 128 x 128; 64 contraction rows per stage
constexpr int kStages = 4, kStageBytes = 32768;      // A halves 2 x 8 KB + B halves 2 x 8 KB
constexpr int kConsumerWarps = 8;                    // two warpgroups, 64 output rows each
constexpr int kThreads = 32 * kConsumerWarps + 32;   // + warp 8: TMA producer
constexpr int kSmem = kStages * kStageBytes + 256 + 1024;

struct WgradArgs {
  int M, No, Ko;
  int tiles_n, tiles_k, splits, blocks_per_split;   // blocks of 64 rows
  float* partial;                                    // [splits][No][Ko] fp32
};

__global__ void __launch_bounds__(kThreads, 1)
wgrad_tn_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmX, const WgradArgs args) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* full = bars;               // [kStages]
  uint64_t* empty = bars + kStages;    // [kStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x % (args.tiles_n * args.tiles_k), sp = blockIdx.x / (args.tiles_n * args.tiles_k);
  const int tn = tile / args.tiles_k, tk = tile % args.tiles_k;
  const int total_blocks = (args.M + KB - 1) / KB;
  const int b0 = sp * args.blocks_per_split;
  const int b1 = min(total_blocks, b0 + args.blocks_per_split);
  const int nblk = max(b1 - b0, 0);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmY), tma_prefetch_desc(&tmX);
    for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1), mbar_init(&empty[s], kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (lane == 0) {
      int slot = 0;
      uint32_t ph = 0;
      for (int b = 0; b < nblk; ++b) {
        mbar_wait(&empty[slot], ph ^ 1);
        mbar_arrive_expect_tx(&full[slot], kStageBytes);
        uint8_t* st = smem + slot * kStageBytes;
        const int row = (b0 + b) * KB;
        // boxes of [64 rows x 64 columns]; columns beyond No / Ko and rows beyond M are zero-filled by TMA
        tma_load_2d(st, &tmY, &full[slot], tn * BM, row);
        tma_load_2d(st + 8192, &tmY, &full[slot], tn * BM + 64, row);
        tma_load_2d(st + 16384, &tmX, &full[slot], tk * BN, row);
        tma_load_2d(st + 24576, &tmX, &full[slot], tk * BN + 64, row);
        if (++slot == kStages) slot = 0, ph ^= 1;
      }
    }
  } else {
    const int wg = warp >> 2;  // output rows [64 wg, 64 wg + 64) of the tile = the wg-th 64-column box of dY
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;   // a split with no rows contributes zeros
    int slot = 0, prev = -1;
    uint32_t ph = 0;
    for (int b = 0; b < nblk; ++b) {
      mbar_wait(&full[slot], ph);
      const uint32_t st = smem_u32(smem + slot * kStageBytes);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KB / 16; ++ks) {
        const uint64_t ad = wgmma_desc_sw128(st + wg * 8192 + ks * 2048);
        const uint64_t bd = wgmma_desc_sw128(st + 16384 + ks * 2048, 8192);
        wgmma_ss<1, 1>(acc, ad, bd, 1u);   // A and B both MN-major
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = slot;
      if (++slot == kStages) slot = 0, ph ^= 1;
    }
    wgmma_wait<0>();
    // ------------------------------------------------------------------ epilogue: accumulators -> fp32 partial tile
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = tn * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2) + h * 8;
      if (r >= args.No) continue;
      float* prow = args.partial + ((size_t)sp * args.No + r) * args.Ko;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = tk * BN + j * 8 + (lane & 3) * 2;   // Ko % 4 == 0: a column pair is inside or outside together
        if (col < args.Ko) *reinterpret_cast<float2*>(prow + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int splits, long n, float* __restrict__ out, int accumulate) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = accumulate ? out[i] : 0.f;
  for (int s = 0; s < splits; ++s) acc += partial[(size_t)s * n + i];
  out[i] = acc;
}

}  // namespace

// fp32 scratch for `splits` partial copies of the [No, Ko] result (wgrad_tn sizes the split count itself: pass the result)
int wgrad_tn_splits(int M, int No, int Ko) {
  const int tiles = ((No + BM - 1) / BM) * ((Ko + BN - 1) / BN);
  const int blocks = (M + KB - 1) / KB;
  int splits = device_sm_count() / tiles;   // one wave of CTAs (129 KB of shared memory each: one CTA per SM)
  if (splits > blocks) splits = blocks;
  if (splits > 64) splits = 64;
  return splits < 1 ? 1 : splits;
}
size_t wgrad_tn_workspace_bytes(int M, int No, int Ko) { return (size_t)wgrad_tn_splits(M, No, Ko) * No * Ko * sizeof(float); }

// dy [M, ld_dy] (No columns used), x [M, ld_x] (Ko columns used), both bf16 row-major with 16-byte aligned rows; out fp32
// [No, Ko] contiguous.  ws: wgrad_tn_workspace_bytes(M, No, Ko).
void wgrad_tn(const bf16* dy, int ld_dy, const bf16* x, int ld_x, int M, int No, int Ko, float* out, int accumulate, void* ws,
              size_t ws_bytes, cudaStream_t stream) {
  N1_CHECK(dy && x && out && ws && M > 0 && No > 0 && Ko > 0, "wgrad_tn: bad arguments");
  N1_CHECK(ld_dy % 8 == 0 && ld_x % 8 == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0,
           "wgrad_tn: operand rows must be 16-byte aligned");
  N1_CHECK(ws_bytes >= wgrad_tn_workspace_bytes(M, No, Ko), "wgrad_tn: workspace too small");
  N1_CHECK((reinterpret_cast<uintptr_t>(ws) & 15) == 0 && Ko % 4 == 0, "wgrad_tn: workspace alignment / Ko % 4");
  static bool attr = false;
  if (!attr) {
    N1_CUDA(cudaFuncSetAttribute(wgrad_tn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    attr = true;
  }
  WgradArgs a;
  a.M = M, a.No = No, a.Ko = Ko;
  a.tiles_n = (No + BM - 1) / BM, a.tiles_k = (Ko + BN - 1) / BN;
  a.splits = wgrad_tn_splits(M, No, Ko);
  const int blocks = (M + KB - 1) / KB;
  a.blocks_per_split = (blocks + a.splits - 1) / a.splits;
  a.partial = static_cast<float*>(ws);
  CUtensorMap tmY = tma_map_2d(dy, M, No, ld_dy, KB, 64, true);
  CUtensorMap tmX = tma_map_2d(x, M, Ko, ld_x, KB, 64, true);
  const int ticket = prof_begin(2.0 * M * (double)No * Ko, No, Ko, M, stream);
  wgrad_tn_kernel<<<a.tiles_n * a.tiles_k * a.splits, kThreads, kSmem, stream>>>(tmY, tmX, a);
  prof_end(ticket, stream);
  prof_count_gemm(2.0 * M * (double)No * Ko);
  N1_CUDA(cudaGetLastError());
  const long n = (long)No * Ko;
  wgrad_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(a.partial, a.splits, n, out, accumulate);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

}  // namespace n1
