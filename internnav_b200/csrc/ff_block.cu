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
//                   2 x 48 KB ring (one [384 x 64] k-block per slot).
//   warpgroups 0-1  consumers, both on the same 64 rows.  The 384-thread kernel is compiled for 168 registers per thread;
//                   the producer warpgroup gives registers back (40) and the consumers take 232 each (setmaxnreg), and
//                   ptxas reports 0 bytes of spill:
//       prologue    x rows -> LayerNorm -> bf16 A operand in shared memory (128-byte swizzled K-major, 48 KB;
//                   dec_tile.cuh holds the LayerNorm, the K = 384 ring loop and the residual epilogue);
//       per hidden chunk of 128 columns: warpgroup g computes its 64 columns  H = LN(x) · W1[128 j + 64 g ..]^T  (wgmma
//                   m64n64k16, fp32 registers), adds b1, GELU, and writes them as bf16 into the swizzled chunk buffer
//                   (double buffered); after one barrier both read the whole chunk back as the A operand of
//                   y[:, 192 g .. 192 g + 192] += GELU(H) · W2[192 g .., chunk]^T  (m64n192k16: the output columns are
//                   split over the warpgroups, 96 accumulator registers each).  GEMM2 of chunk j stays in flight under
//                   GEMM1 of chunk j + 1, and one warpgroup's GELU runs under the other's MMAs;
//       epilogue    y + x + b2 -> bf16 -> global (in place: a thread re-reads exactly the elements it overwrites).
#include <mutex>

#include "dec_tile.cuh"

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

__global__ void __launch_bounds__(kThreads, 1)
ff_block_kernel(const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2, const FfArgs args) {
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
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW1), tma_prefetch_desc(&tmW2);
    for (int s = 0; s < kS1; ++s) mbar_init(&w1_full[s], 1), mbar_init(&w1_empty[s], kConsumerWarps);
    for (int s = 0; s < kS2; ++s) mbar_init(&w2_full[s], 1), mbar_init(&w2_empty[s], kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      // ------------------------------------------------------------------ TMA producer of W1 (GEMM1's ring)
      Ring<kS1> r;
      for (int t = blockIdx.x; t < args.tiles_m; t += gridDim.x)
        for (int j = 0; j < NCH; ++j)
          for (int kb = 0; kb < D / 64; ++kb) {  // W1 rows [128j, 128j+128), k-block kb
            mbar_wait(&w1_empty[r.slot], r.phase ^ 1);
            mbar_arrive_expect_tx(&w1_full[r.slot], kS1Bytes);
            tma_load_2d(sW1 + r.slot * kS1Bytes, &tmW1, &w1_full[r.slot], kb * 64, j * HC);
            r.advance();
          }
    } else if (warp == kConsumerWarps + 1 && lane == 0) {
      // ------------------------------------------------------------------ TMA producer of W2 (GEMM2's ring)
      Ring<kS2> r;
      for (int t = blockIdx.x; t < args.tiles_m; t += gridDim.x)
        for (int j = 0; j < NCH; ++j)
          for (int kb = 0; kb < HC / 64; ++kb) {  // W2[:, 128j + 64kb : +64) as two boxes of 192 output rows
            mbar_wait(&w2_empty[r.slot], r.phase ^ 1);
            mbar_arrive_expect_tx(&w2_full[r.slot], kS2Bytes);
            uint8_t* dst = sW2 + r.slot * kS2Bytes;
            tma_load_2d(dst, &tmW2, &w2_full[r.slot], j * HC + kb * 64, 0);
            tma_load_2d(dst + kS2Bytes / 2, &tmW2, &w2_full[r.slot], j * HC + kb * 64, 192);
            r.advance();
          }
    }
  } else {
    // ------------------------------------------------------------------ 2 consumer warpgroups
    setmaxnreg_inc<kConsumerRegs>();
    const int cw = warp;                     // 0..7
    const int g = cw >> 2;                   // warpgroup: hidden columns [64 g, +64) of a chunk, output columns [192 g, +192)
    const int quad = lane & 3;
    const int r0 = (cw & 3) * 16 + (lane >> 2);  // this thread's accumulator rows: r0 and r0 + 8
    Ring<kS1> r1;
    Ring<kS2> r2;
    for (int tm = blockIdx.x; tm < args.tiles_m; tm += gridDim.x) {
      const long row0 = (long)tm * BM;
      // every MMA of the previous tile has completed in both warpgroups: the A operand and the chunk buffers are free
      consumer_barrier();
      ln384_to_tile<true>(sA, args.x, args.ldx, row0, args.M - tm * BM, args.ln_w, args.ln_b, args.eps, cw, lane);
      fence_proxy_async_smem();
      consumer_barrier();

      // Zeroed although the first MMA overwrites it: the accumulator is an in-out operand of every wgmma, and without a
      // definition here it would count as live through the LayerNorm prologue above (96 registers, which then spills).
      float y[96] = {};
      for (int j = 0; j < NCH; ++j) {
        // ---- GEMM1(j): this warpgroup's 64 hidden columns, K = 384: 6 k-blocks x 4 k-steps of m64n64k16.  Once the first
        // k-block's wait has seen GEMM2(j - 1) complete, its two W2 slots are released.
        float h[32];
        mma_k384(h, sA, sW1, w1_full, w1_empty, r1, kS1Bytes, g * 8192, lane, [&] {
          if (lane == 0 && j > 0) {
            mbar_arrive(&w2_empty[r2.slot]);
            mbar_arrive(&w2_empty[r2.slot ^ 1]);
          }
        });
        // ---- + b1, GELU, bf16 -> chunk buffer j % 2 (k-block g: its 64 columns are this warpgroup's)
        uint8_t* hb = sH + (j & 1) * kHBytes;
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
            for (int hh = 0; hh < 2; ++hh)
              *reinterpret_cast<uint32_t*>(hb + sw128_offset(r0 + hh * 8, g * 64 + (jj + u) * 8 + quad * 2)) =
                  pack_bf16(v[4 * u + 2 * hh], v[4 * u + 2 * hh + 1]);
        }
        fence_proxy_async_smem();
        // The other warpgroup passed this barrier for chunk j - 1 only after its GEMM2(j - 2) had completed, so buffer
        // j % 2 was free when it was written above; now both halves of chunk j are visible.
        consumer_barrier();
        // ---- GEMM2(j): y[:, 192 g ..] += GELU(H_j) · W2[192 g .., chunk]^T, K = 128: 2 k-blocks x 4 k-steps of m64n192k16
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < HC / 64; ++kb) {
          mbar_wait(&w2_full[r2.slot], r2.phase);
          const uint64_t ad = wgmma_desc_sw128(smem_u32(hb + kb * 8192));
          const uint64_t bd = wgmma_desc_sw128(smem_u32(sW2 + r2.slot * kS2Bytes + g * (kS2Bytes / 2)));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(y, ad + 2 * k, bd + 2 * k, (j | kb | k) != 0 ? 1u : 0u);
          r2.advance();
        }
        wgmma_commit();
      }
      wgmma_wait<0>();
      if (lane == 0) {
        mbar_arrive(&w2_empty[r2.slot]);
        mbar_arrive(&w2_empty[r2.slot ^ 1]);
      }
      // ---- epilogue: out = y + x + b2
      residual_epilogue_192<true>(y, args.x, args.ldx, args.out, args.ldo, args.b2, row0, args.M - tm * BM, g, r0, quad);
    }
  }
}

void launch_ff(const bf16* w1, const bf16* w2, const FfArgs& a, cudaStream_t stream) {
  static std::once_flag once;
  std::call_once(once, [] { cudaFuncSetAttribute(ff_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem); });
  const CUtensorMap tmW1 = tma_map_2d(w1, F, D, D, HC, 64, true);
  const CUtensorMap tmW2 = tma_map_2d(w2, D, F, F, 192, 64, true);
  const int sms = device_sm_count();
  const int grid = a.tiles_m < sms ? a.tiles_m : sms;
  const int ticket = prof_begin(4.0 * a.M * (double)D * F, a.M, -F, D, stream);  // N = -1536 marks the fused FF block
  ff_block_kernel<<<grid, kThreads, kSmem, stream>>>(tmW1, tmW2, a);
  prof_end(ticket, stream);
  prof_count_gemm(4.0 * a.M * (double)D * F);
  N1_CUDA(cudaGetLastError());
}

}  // namespace

// x [M, ldx] bf16 residual stream (read), out [M, ldo] bf16 (written; may alias x); w1 [1536, 384], w2 [384, 1536] bf16
// contiguous; ln_w / ln_b / b2 fp32 [384], b1 fp32 [1536].  out = x + W2 GELU(W1 LN(x) + b1) + b2.
void ff_block_384(const bf16* x, int ldx, const float* ln_w, const float* ln_b, float eps, const bf16* w1, const float* b1,
                  const bf16* w2, const float* b2, bf16* out, int ldo, int M, cudaStream_t stream) {
  if (M <= 0) return;
  N1_CHECK(x && out && w1 && w2 && ln_w && ln_b && b1 && b2, "ff_block_384: null pointer");
  N1_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0 && ldx % 8 == 0, "ff_block_384: misaligned x");
  N1_CHECK((reinterpret_cast<uintptr_t>(out) & 3) == 0 && ldo % 2 == 0, "ff_block_384: misaligned out");
  FfArgs a;
  a.M = M, a.tiles_m = (M + BM - 1) / BM;
  a.x = x, a.ldx = ldx, a.ln_w = ln_w, a.ln_b = ln_b, a.eps = eps, a.b1 = b1, a.b2 = b2, a.out = out, a.ldo = ldo;
  launch_ff(w1, w2, a, stream);
}

}  // namespace n1
