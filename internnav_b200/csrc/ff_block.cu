// FF block of the NavDP decoder layer as ONE kernel, hidden activations never leaving the SM:
//
//     x  <-  x + W2 · GELU(W1 · LayerNorm(x) + b1) + b2            (D = 384, F = 1536; navdp.py L57-66: norm3 / linear1 /
//                                                                    exact GELU / linear2 / residual of the pre-norm layer)
//
// replaces three launches (LayerNorm, FF1+GELU GEMM, FF2+residual GEMM) and the HBM round trips of the [rows, 384]
// normalised input and the [rows, 1536] hidden.  Per CTA, one 64-row tile at a time (persistent over tiles):
//
//   warpgroup 2     producers (warps 10, 11 only hand their registers over and leave): warp 8 streams W1 through a
//                   3 x 16 KB ring (one [128 x 64] k-block of a hidden chunk per slot), warp 9 streams W2 through a
//                   2 x 48 KB ring (one [384 x 64] k-block per slot).  CM = 2: the two CTAs of a cluster work on
//                   neighbouring row tiles, fetch half of every slot each and multicast it.
//   warpgroups 0-1  consumers, both on the same 64 rows.  The 384-thread kernel is compiled for 168 registers per thread;
//                   the producer warpgroup gives registers back (40) and the consumers take 232 each (setmaxnreg), and
//                   ptxas reports 0 bytes of spill for both cluster variants:
//       prologue    x rows -> LayerNorm -> bf16 A operand in shared memory (128-byte swizzled K-major, 48 KB);
//       per hidden chunk of 128 columns: warpgroup g computes its 64 columns  H = LN(x) · W1[128 j + 64 g ..]^T  (wgmma
//                   m64n64k16, fp32 registers), adds b1, GELU, and writes them as bf16 into the swizzled chunk buffer
//                   (double buffered); after one barrier both read the whole chunk back as the A operand of
//                   y[:, 192 g .. 192 g + 192] += GELU(H) · W2[192 g .., chunk]^T  (m64n192k16: the output columns are
//                   split over the warpgroups, 96 accumulator registers each).  GEMM2 of chunk j stays in flight under
//                   GEMM1 of chunk j + 1, and one warpgroup's GELU runs under the other's MMAs;
//       epilogue    y + x + b2 -> bf16 -> global (in place: a thread re-reads exactly the elements it overwrites).
#include <stdlib.h>

#include <mutex>

#include "n1_ops.h"
#include "n1_ptx.cuh"

namespace n1 {
namespace {

constexpr int D = 384, F = 1536, BM = 64, HC = 128;
constexpr int NCH = F / HC;                          // 12 hidden chunks
constexpr int kS1 = 3, kS1Bytes = HC * 64 * 2;       // W1 ring: one k-block [128 x 64] of a hidden chunk per slot
constexpr int kS2 = 2, kS2Bytes = D * 64 * 2;        // W2 ring: one k-block [384 x 64] of a hidden chunk per slot
constexpr int kABytes = BM * D * 2;                  // 49152: 6 k-blocks of [64 x 64]
constexpr int kHBytes = BM * HC * 2;                 // 16384: one GELU(H) chunk, 2 k-blocks of [64 x 64]
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 128;  // 384: the producers are a whole warpgroup (setmaxnreg)
constexpr int kSmem = kABytes + 2 * kHBytes + kS1 * kS1Bytes + kS2 * kS2Bytes + 256 + 1024;
static_assert(kSmem <= 232448, "ff_block: shared memory budget (227 KB per block)");

struct FfArgs {
  int M;
  int tiles_m;
  const bf16* x;   // [M, ldx] residual stream in
  int ldx;
  const float* ln_w;
  const float* ln_b;
  float eps;
  const float* b1;
  const float* b2;
  bf16* out;
  int ldo;
};

// barrier among the consumer warps only (named barrier 1; the producer warps never join it)
__device__ __forceinline__ void consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerWarps * 32) : "memory"); }

template <int CM>
__global__ void __launch_bounds__(kThreads, 1)
ff_block_kernel(const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2, const FfArgs args) {
  constexpr uint16_t kMask = (1u << CM) - 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sH = smem + kABytes;
  uint8_t* sW1 = sH + 2 * kHBytes;
  uint8_t* sW2 = sW1 + kS1 * kS1Bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sW2 + kS2 * kS2Bytes);
  uint64_t* w1_full = bars;                // [3]
  uint64_t* w1_empty = bars + 3;           // [3]
  uint64_t* w2_full = bars + 6;            // [2]
  uint64_t* w2_empty = bars + 8;           // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = CM > 1 ? (int)cluster_ctarank() : 0;
  const int cluster_id = blockIdx.x / CM, num_clusters = gridDim.x / CM;
  const int super_m = (args.tiles_m + CM - 1) / CM;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW1), tma_prefetch_desc(&tmW2);
    // every consumer warp of every CTA of the cluster releases a slot (its halves live in all of them)
    for (int s = 0; s < kS1; ++s) mbar_init(&w1_full[s], 1), mbar_init(&w1_empty[s], kConsumerWarps * CM);
    for (int s = 0; s < kS2; ++s) mbar_init(&w2_full[s], 1), mbar_init(&w2_empty[s], kConsumerWarps * CM);
    fence_mbar_init();
  }
  // peers' barriers must be initialised before any multicast / remote arrive reaches them
  if (CM > 1) cluster_sync_all(); else __syncthreads();

  if (warp >= kConsumerWarps) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      // ------------------------------------------------------------------ TMA producer of W1 (GEMM1's ring)
      int slot = 0;
      uint32_t ph = 0;
      for (int t = cluster_id; t < super_m; t += num_clusters)
        for (int j = 0; j < NCH; ++j)
          for (int kb = 0; kb < D / 64; ++kb) {  // W1 rows [128j, 128j+128), k-block kb
            mbar_wait(&w1_empty[slot], ph ^ 1);
            mbar_arrive_expect_tx(&w1_full[slot], kS1Bytes);
            uint8_t* dst = sW1 + slot * kS1Bytes;
            if (CM == 1) {
              tma_load_2d(dst, &tmW1, &w1_full[slot], kb * 64, j * HC);
            } else {  // each CTA fetches 64 of the 128 rows and multicasts them
              tma_load_2d_mc(dst + rank * (kS1Bytes / 2), &tmW1, &w1_full[slot], kb * 64, j * HC + rank * (HC / 2), kMask);
            }
            if (++slot == kS1) slot = 0, ph ^= 1;
          }
    } else if (warp == kConsumerWarps + 1 && lane == 0) {
      // ------------------------------------------------------------------ TMA producer of W2 (GEMM2's ring)
      int slot = 0;
      uint32_t ph = 0;
      for (int t = cluster_id; t < super_m; t += num_clusters)
        for (int j = 0; j < NCH; ++j)
          for (int kb = 0; kb < HC / 64; ++kb) {  // W2[:, 128j + 64kb : +64) as two boxes of 192 output rows
            mbar_wait(&w2_empty[slot], ph ^ 1);
            mbar_arrive_expect_tx(&w2_full[slot], kS2Bytes);
            uint8_t* dst = sW2 + slot * kS2Bytes;
            if (CM == 1) {
              tma_load_2d(dst, &tmW2, &w2_full[slot], j * HC + kb * 64, 0);
              tma_load_2d(dst + kS2Bytes / 2, &tmW2, &w2_full[slot], j * HC + kb * 64, 192);
            } else {
              tma_load_2d_mc(dst + rank * (kS2Bytes / 2), &tmW2, &w2_full[slot], j * HC + kb * 64, rank * 192, kMask);
            }
            if (++slot == kS2) slot = 0, ph ^= 1;
          }
    }
  } else {
    // ------------------------------------------------------------------ 2 consumer warpgroups
    setmaxnreg_inc<kConsumerRegs>();
    const int cw = warp;                     // 0..7
    const int g = cw >> 2;                   // warpgroup: hidden columns [64 g, +64) of a chunk, output columns [192 g, +192)
    const int quad = lane & 3;
    const int r0 = (cw & 3) * 16 + (lane >> 2);  // this thread's accumulator rows: r0 and r0 + 8
    auto release = [&](uint64_t* bar) {      // called by lane 0 of every consumer warp
      if (CM == 1) {
        mbar_arrive(bar);
      } else {
#pragma unroll
        for (int c = 0; c < CM; ++c) mbar_arrive_cluster(bar, c);
      }
    };
    int s1 = 0, s2 = 0;
    uint32_t ph1 = 0, ph2 = 0;
    for (int t = cluster_id; t < super_m; t += num_clusters) {
      const int tm = t * CM + rank;
      // every MMA of the previous tile has completed in both warpgroups: the A operand and the chunk buffers are free
      consumer_barrier();
      // ---- prologue: LayerNorm, one warp per row (8 rows per warp), coalesced 8-byte loads, two-pass variance.  All 24
      // loads of the warp's 8 rows are issued before the first use and the shuffle reductions advance in lock-step.
      {
        uint2 q[8][3];
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
          const long grow = (long)tm * BM + cw * 8 + rr;
          const bf16* xr = args.x + grow * args.ldx;
#pragma unroll
          for (int i = 0; i < 3; ++i)
            q[rr][i] = grow < args.M ? __ldg(reinterpret_cast<const uint2*>(xr + (lane + i * 32) * 4)) : make_uint2(0u, 0u);
        }
        float s[8], sq[8];
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
          s[rr] = 0.f;
#pragma unroll
          for (int i = 0; i < 3; ++i)
            s[rr] += bf16_lo(q[rr][i].x) + bf16_hi(q[rr][i].x) + bf16_lo(q[rr][i].y) + bf16_hi(q[rr][i].y);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) s[rr] += __shfl_xor_sync(0xffffffffu, s[rr], o);
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
          const float mu = s[rr] * (1.0f / D);
          s[rr] = mu;
          sq[rr] = 0.f;
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            const float a = bf16_lo(q[rr][i].x) - mu, b = bf16_hi(q[rr][i].x) - mu;
            const float c = bf16_lo(q[rr][i].y) - mu, d = bf16_hi(q[rr][i].y) - mu;
            sq[rr] += a * a + b * b + c * c + d * d;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) sq[rr] += __shfl_xor_sync(0xffffffffu, sq[rr], o);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int col = (lane + i * 32) * 4;
          const float4 lw = __ldg(reinterpret_cast<const float4*>(args.ln_w + col));
          const float4 lb = __ldg(reinterpret_cast<const float4*>(args.ln_b + col));
          // K-major, 128-byte swizzle: k-block col / 64, 16-byte chunk (col % 64) / 8 at position chunk ^ (row % 8)
          const int kb = col >> 6, ch = (col & 63) >> 3;
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) {
            const float mu = s[rr], rstd = rsqrtf(sq[rr] * (1.0f / D) + args.eps);
            const float y0 = (bf16_lo(q[rr][i].x) - mu) * rstd * lw.x + lb.x, y1 = (bf16_hi(q[rr][i].x) - mu) * rstd * lw.y + lb.y;
            const float y2 = (bf16_lo(q[rr][i].y) - mu) * rstd * lw.z + lb.z, y3 = (bf16_hi(q[rr][i].y) - mu) * rstd * lw.w + lb.w;
            // row cw * 8 + rr: 8-row group cw, row rr inside it
            uint8_t* dst = sA + kb * 8192 + cw * 1024 + rr * 128 + ((ch ^ rr) << 4) + (col & 7) * 2;
            *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
          }
        }
      }
      fence_proxy_async_smem();
      consumer_barrier();

      // Zeroed although the first MMA overwrites it: the accumulator is an in-out operand of every wgmma, and without a
      // definition here it would count as live through the LayerNorm prologue above (96 registers, which then spills).
      float y[96] = {};
      for (int j = 0; j < NCH; ++j) {
        // ---- GEMM1(j): this warpgroup's 64 hidden columns, K = 384: 6 k-blocks x 4 k-steps of m64n64k16
        float h[32];
        int prev1 = -1;
#pragma unroll 1
        for (int kb = 0; kb < D / 64; ++kb) {
          mbar_wait(&w1_full[s1], ph1);
          const uint64_t ad = wgmma_desc_sw128(smem_u32(sA + kb * 8192));
          const uint64_t bd = wgmma_desc_sw128(smem_u32(sW1 + s1 * kS1Bytes + g * 8192));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(h, ad + 2 * k, bd + 2 * k, (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();  // everything before this k-block is complete: GEMM2(j - 1) (kb == 0) or k-block kb - 1
          if (lane == 0) {
            if (kb == 0 && j > 0) {  // the two W2 slots of GEMM2(j - 1)
              release(&w2_empty[s2]);
              release(&w2_empty[s2 ^ 1]);
            }
            if (prev1 >= 0) release(&w1_empty[prev1]);
          }
          prev1 = s1;
          if (++s1 == kS1) s1 = 0, ph1 ^= 1;
        }
        wgmma_wait<0>();
        if (lane == 0) release(&w1_empty[prev1]);
        // ---- + b1, GELU, bf16 -> chunk buffer j % 2 (k-block g: its 64 columns are this warpgroup's)
        uint8_t* hb = sH + (j & 1) * kHBytes + g * 8192;
#pragma unroll
        for (int jj = 0; jj < 8; jj += 2) {
          float v[8];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float2 b = __ldg(reinterpret_cast<const float2*>(args.b1 + j * HC + g * 64 + (jj + u) * 8 + quad * 2));
            v[4 * u + 0] = h[(jj + u) * 4 + 0] + b.x, v[4 * u + 1] = h[(jj + u) * 4 + 1] + b.y;
            v[4 * u + 2] = h[(jj + u) * 4 + 2] + b.x, v[4 * u + 3] = h[(jj + u) * 4 + 3] + b.y;
          }
          gelu_erf8(v);
#pragma unroll
          for (int u = 0; u < 2; ++u)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int r = r0 + hh * 8;
              // column 8 (jj + u) + 2 quad of the k-block: 16-byte chunk jj + u at position chunk ^ (row % 8)
              *reinterpret_cast<uint32_t*>(hb + (r >> 3) * 1024 + (r & 7) * 128 + (((jj + u) ^ (r & 7)) << 4) + quad * 4) =
                  pack_bf16(v[4 * u + 2 * hh], v[4 * u + 2 * hh + 1]);
            }
        }
        fence_proxy_async_smem();
        // The other warpgroup passed this barrier for chunk j - 1 only after its GEMM2(j - 2) had completed, so buffer
        // j % 2 was free when it was written above; now both halves of chunk j are visible.
        consumer_barrier();
        // ---- GEMM2(j): y[:, 192 g ..] += GELU(H_j) · W2[192 g .., chunk]^T, K = 128: 2 k-blocks x 4 k-steps of m64n192k16
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < HC / 64; ++kb) {
          mbar_wait(&w2_full[s2], ph2);
          const uint64_t ad = wgmma_desc_sw128(smem_u32(sH + (j & 1) * kHBytes + kb * 8192));
          const uint64_t bd = wgmma_desc_sw128(smem_u32(sW2 + s2 * kS2Bytes + g * (kS2Bytes / 2)));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(y, ad + 2 * k, bd + 2 * k, (j | kb | k) != 0 ? 1u : 0u);
          if (++s2 == kS2) s2 = 0, ph2 ^= 1;
        }
        wgmma_commit();
      }
      wgmma_wait<0>();
      if (lane == 0) {
        release(&w2_empty[s2]);
        release(&w2_empty[s2 ^ 1]);
      }
      // ---- epilogue: out = y + x + b2
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const long row = (long)tm * BM + r0 + hh * 8;
        if (row >= args.M) continue;
        const bf16* xr = args.x + row * args.ldx + g * 192 + quad * 2;
        bf16* orow = args.out + row * args.ldo + g * 192 + quad * 2;
#pragma unroll
        for (int jj = 0; jj < 24; ++jj) {
          const uint32_t xv = __ldg(reinterpret_cast<const uint32_t*>(xr + jj * 8));
          const float2 b = __ldg(reinterpret_cast<const float2*>(args.b2 + g * 192 + jj * 8 + quad * 2));
          *reinterpret_cast<uint32_t*>(orow + jj * 8) =
              pack_bf16(y[jj * 4 + 2 * hh] + bf16_lo(xv) + b.x, y[jj * 4 + 2 * hh + 1] + bf16_hi(xv) + b.y);
        }
      }
    }
  }
  // no CTA may retire while a peer can still multicast into it or arrive on its barriers
  if (CM > 1) cluster_sync_all();
}

template <int CM>
void launch_ff(const bf16* w1, const bf16* w2, const FfArgs& a, cudaStream_t stream) {
  static std::once_flag once;
  static int max_clusters = 0;
  std::call_once(once, [] {
    cudaFuncSetAttribute(ff_block_kernel<CM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    max_clusters = device_sm_count() / CM;
    if (CM > 1) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(device_sm_count() / CM * CM), cfg.blockDim = dim3(kThreads), cfg.dynamicSmemBytes = kSmem;
      cudaLaunchAttribute at;
      at.id = cudaLaunchAttributeClusterDimension;
      at.val.clusterDim.x = CM, at.val.clusterDim.y = 1, at.val.clusterDim.z = 1;
      cfg.attrs = &at, cfg.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, ff_block_kernel<CM>, &cfg) == cudaSuccess && n > 0) max_clusters = n;
    }
  });
  CUtensorMap tmW1 = tma_map_2d(w1, F, D, D, HC / CM, 64, true);
  CUtensorMap tmW2 = tma_map_2d(w2, D, F, F, 192, 64, true);
  const int super_m = (a.tiles_m + CM - 1) / CM;
  const int clusters = super_m < max_clusters ? super_m : max_clusters;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(clusters * CM), cfg.blockDim = dim3(kThreads), cfg.dynamicSmemBytes = kSmem, cfg.stream = stream;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeClusterDimension;
  at.val.clusterDim.x = CM, at.val.clusterDim.y = 1, at.val.clusterDim.z = 1;
  cfg.attrs = &at, cfg.numAttrs = 1;
  const int ticket = prof_begin(4.0 * a.M * (double)D * F, a.M, -F, D, stream);  // N = -1536 marks the fused FF block
  N1_CUDA(cudaLaunchKernelEx(&cfg, ff_block_kernel<CM>, tmW1, tmW2, a));
  prof_end(ticket, stream);
  prof_count_gemm(4.0 * a.M * (double)D * F);
  N1_CUDA(cudaGetLastError());
}

}  // namespace

// x [M, ldx] bf16 residual stream (read), out [M, ldo] bf16 (written; may alias x); w1 [1536, 384], w2 [384, 1536] bf16
// contiguous; ln_w / ln_b / b2 fp32 [384], b1 fp32 [1536].  out = x + W2 GELU(W1 LN(x) + b1) + b2.
void ff_block_384(const bf16* x, int ldx, const float* ln_w, const float* ln_b, float eps, const bf16* w1, const float* b1,
                  const bf16* w2, const float* b2, bf16* out, int ldo, int M, int cluster, cudaStream_t stream) {
  if (M <= 0) return;
  N1_CHECK(x && out && w1 && w2 && ln_w && ln_b && b1 && b2, "ff_block_384: null pointer");
  N1_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0 && ldx % 8 == 0, "ff_block_384: misaligned x");
  N1_CHECK((reinterpret_cast<uintptr_t>(out) & 3) == 0 && ldo % 2 == 0, "ff_block_384: misaligned out");
  FfArgs a;
  a.M = M, a.tiles_m = (M + BM - 1) / BM;
  a.x = x, a.ldx = ldx, a.ln_w = ln_w, a.ln_b = ln_b, a.eps = eps, a.b1 = b1, a.b2 = b2, a.out = out, a.ldo = ldo;
  if (cluster >= 2 && a.tiles_m >= 2) launch_ff<2>(w1, w2, a, stream);
  else launch_ff<1>(w1, w2, a, stream);
}

}  // namespace n1
