// Self- and cross-attention sublayers of the NavDP decoder layer, each as ONE kernel (navdp.py L57-66, pre-norm layer):
//
//     self:   x  <-  x + W_o · MHA_causal(q, k, v = LN1(x) · W_qkv^T + b_qkv) + b_o       (keys: the row's own trajectory)
//     cross:  x  <-  x + W_o · MHA(LN2(x) · W_q^T + b_q, K_env, V_env) + b_o              (keys: the env's Mtok <= 64 rows)
//
// with D = 384, 8 heads of dim 48.  Each replaces LayerNorm + projection GEMM + attention + output GEMM with residual, and
// the HBM round trips of the normalised rows, q / k / v and the attention output.  Both sublayers are local to a row tile:
// a tile is floor(64 / T) whole trajectories of ONE environment (an environment's last tile may hold fewer), so
// self-attention never looks outside the tile and cross-attention reads one environment's projected condition K / V.
// Per CTA (persistent over tiles), the skeleton of ff_block.cu:
//
//   warpgroup 2     producer (warp 8, one lane; the other producer warps only hand their registers over): streams every
//                   weight k-block of the tile through one 2 x 48 KB TMA ring -- first 4 head pairs x 6 k-blocks of the
//                   input projection (slot = [q_h | k_h | v_h] rows of head h for warpgroup 0 and of head h + 4 for
//                   warpgroup 1, 2 x 144 x 64 for self, 2 x 48 x 64 for cross), then 6 k-blocks [384 x 64] of W_o.
//   warpgroups 0-1  consumers at 232 registers, both on the same rows; warpgroup g owns heads 4 g .. 4 g + 3:
//       prologue    x rows -> LayerNorm -> bf16 A operand (128-byte swizzled K-major, 48 KB), as in ff_block.cu (the
//                   LayerNorm, the K = 384 ring loop, the attention core and the epilogue are in dec_tile.cuh);
//       per head    projection of the head (wgmma m64n144k16 / m64n48k16, fp32), + bias, bf16.  Q stays in registers: the
//                   accumulator layout of wgmma is the A-fragment layout of mma.sync.  K and V go to the warpgroup's
//                   staging buffer (self: from the accumulators; cross: the environment's rows of the layer's K / V).
//                   Each warp then runs S = Q K^T over 64 keys, the masked softmax (fp32, P rounded to bf16) and O = P V
//                   on mma.sync.m16n8k16 for its 16 rows, with attn_small_kernel's (attention.cu) code, and writes
//                   O / rowsum as bf16 into the swizzled O tile;
//       epilogue    y[:, 192 g ..] = O · W_o[192 g ..]^T (m64n192k16, output columns split over the warpgroups),
//                   x = y + b_o + x -> bf16, in place (a thread re-reads exactly the elements it overwrites).
//
// Shared memory (bytes): LN tile 49152 | O tile 49152 | ring 2 x 49152 | K / V staging 2 warpgroups x 2 x 64 x 112
// (rows padded from 96 to 112 bytes: conflict-free ldmatrix) | 6 mbarriers.  226 560 with the 1024-byte alignment slack.
#include <mutex>

#include "dec_tile.cuh"

namespace n1 {
namespace {

constexpr int D = 384, HD = 48, BM = 64;
constexpr int kABytes = BM * D * 2;             // 49152: 6 k-blocks of [64 x 64]
constexpr int kSlots = 2, kSlotBytes = D * 64 * 2;  // one W_o k-block [384 x 64]; an input-projection k-block fits too
constexpr int kKvRow = 112;                     // staging row stride: 48 bf16 + 16 bytes of padding
constexpr int kKvBytes = BM * kKvRow;           // one [64 x 48] K or V buffer
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 128;
constexpr int kSmem = 2 * kABytes + kSlots * kSlotBytes + 2 * 2 * kKvBytes + 256 + 1024;
static_assert(kSmem <= 232448, "dec_attn_block: shared memory budget (227 KB per block)");

struct DecAttnArgs {
  bf16* x;  // [rows, ldx] residual stream, updated in place
  int ldx;
  const float* ln_w;
  const float* ln_b;
  float eps;
  const float* b_in;  // self: in_proj bias [1152] (q | k | v); cross: q bias [384]
  const float* b_o;   // [384]
  const bf16* kv;     // cross: K of environment e, key j at kv[(e * mtok + j) * ldkv + c], V at + 384
  int ldkv;
  int mtok;
  int Ns, T, tpt, tiles_per_env, tiles;  // tpt: trajectories per tile
  int causal;
};

__device__ __forceinline__ void warpgroup_barrier(int g) { asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory"); }

template <bool kSelf>
__global__ void __launch_bounds__(kThreads, 1)
dec_attn_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmO, const DecAttnArgs args) {
  constexpr int NP = kSelf ? 3 * HD : HD;          // projection columns of one head
  constexpr int kHeadBytes = NP * 64 * 2;          // one head's rows of an input-projection k-block
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sO = smem + kABytes;
  uint8_t* sW = sO + kABytes;
  uint8_t* sKV = sW + kSlots * kSlotBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + 4 * kKvBytes);
  uint64_t* full = bars;           // [2]
  uint64_t* empty = bars + kSlots;  // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmIn), tma_prefetch_desc(&tmO);
    for (int s = 0; s < kSlots; ++s) mbar_init(&full[s], 1), mbar_init(&empty[s], kConsumerWarps);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      Ring<kSlots> r;
      for (int t = blockIdx.x; t < args.tiles; t += gridDim.x) {
        for (int hp = 0; hp < 4; ++hp)
          for (int kb = 0; kb < D / 64; ++kb) {
            mbar_wait(&empty[r.slot], r.phase ^ 1);
            mbar_arrive_expect_tx(&full[r.slot], 2 * kHeadBytes);
            uint8_t* dst = sW + r.slot * kSlotBytes;
#pragma unroll
            for (int g = 0; g < 2; ++g) {
              const int h = 4 * g + hp;
#pragma unroll
              for (int part = 0; part < NP / HD; ++part)  // q_h, k_h, v_h rows of the in_proj weight
                tma_load_2d(dst + g * kHeadBytes + part * HD * 128, &tmIn, &full[r.slot], kb * 64, part * D + h * HD);
            }
            r.advance();
          }
        for (int kb = 0; kb < D / 64; ++kb) {
          mbar_wait(&empty[r.slot], r.phase ^ 1);
          mbar_arrive_expect_tx(&full[r.slot], kSlotBytes);
          uint8_t* dst = sW + r.slot * kSlotBytes;
          tma_load_2d(dst, &tmO, &full[r.slot], kb * 64, 0);
          tma_load_2d(dst + kSlotBytes / 2, &tmO, &full[r.slot], kb * 64, 192);
          r.advance();
        }
      }
    }
  } else {
    setmaxnreg_inc<kConsumerRegs>();
    const int cw = warp;                            // 0..7
    const int g = cw >> 2;                          // warpgroup
    const int wtid = threadIdx.x & 127;             // thread within the warpgroup
    const int quad = lane & 3;
    const int r0 = (cw & 3) * 16 + (lane >> 2);     // this thread's accumulator rows: r0 and r0 + 8
    uint8_t* sK = sKV + g * 2 * kKvBytes;
    uint8_t* sV = sK + kKvBytes;
    const float sl2 = 0.14433756729740643f * 1.4426950408889634f;  // 48^-1/2 * log2(e)
    Ring<kSlots> ring;
    for (int t = blockIdx.x; t < args.tiles; t += gridDim.x) {
      const int env = t / args.tiles_per_env;
      const int traj0 = (t - env * args.tiles_per_env) * args.tpt;
      const int ntraj = min(args.tpt, args.Ns - traj0);
      const long row0 = ((long)env * args.Ns + traj0) * args.T;
      const int nrows = ntraj * args.T;
      // every MMA of the previous tile has completed in both warpgroups: the LN and O tiles are free
      consumer_barrier();
      // ---- prologue: LayerNorm; rows past the tile read as zeros
      ln384_to_tile<false>(sA, args.x, args.ldx, row0, nrows, args.ln_w, args.ln_b, args.eps, cw, lane);
      fence_proxy_async_smem();
      consumer_barrier();

      for (int hp = 0; hp < 4; ++hp) {
        const int h = 4 * g + hp;
        // the warpgroup's previous head is done reading the K / V staging buffer
        warpgroup_barrier(g);
        if (!kSelf) {  // this head's K / V rows of the tile's environment; keys past mtok are zeros (and masked)
          const bf16* kb0 = args.kv + (long)env * args.mtok * args.ldkv + h * HD;
          for (int c = wtid; c < 2 * BM * 6; c += 128) {
            const int v = c / (BM * 6), j = (c / 6) % BM, ch = c % 6;
            uint4 val = make_uint4(0u, 0u, 0u, 0u);
            if (j < args.mtok) val = __ldg(reinterpret_cast<const uint4*>(kb0 + (long)j * args.ldkv + v * D + ch * 8));
            *reinterpret_cast<uint4*>((v ? sV : sK) + j * kKvRow + ch * 16) = val;
          }
        }
        // ---- projection of head h: acc[64 x NP] = LN(x) · W_in[head rows]^T, K = 384
        float acc[NP / 2];
        mma_k384(acc, sA, sW, full, empty, ring, kSlotBytes, g * kHeadBytes, lane, [] {});
        // ---- + bias, bf16.  Column 8 j + 2 quad (+1) of acc[4 j ..] is part j / 6 (q, k, v) of the head.
        uint32_t qf[3][4];
#pragma unroll
        for (int j = 0; j < NP / 8; ++j) {
          const int part = j / 6, c = (j % 6) * 8 + quad * 2;
          const float2 b = __ldg(reinterpret_cast<const float2*>(args.b_in + part * D + h * HD + c));
          const uint32_t lo = pack_bf16(acc[4 * j] + b.x, acc[4 * j + 1] + b.y);
          const uint32_t hi = pack_bf16(acc[4 * j + 2] + b.x, acc[4 * j + 3] + b.y);
          if (part == 0) {
            qf[j >> 1][(j & 1) * 2] = lo, qf[j >> 1][(j & 1) * 2 + 1] = hi;
          } else {
            uint8_t* buf = part == 1 ? sK : sV;
            *reinterpret_cast<uint32_t*>(buf + r0 * kKvRow + c * 2) = lo;
            *reinterpret_cast<uint32_t*>(buf + (r0 + 8) * kKvRow + c * 2) = hi;
          }
        }
        warpgroup_barrier(g);  // K / V of head h staged
        // ---- attention of this warp's 16 rows over the 64 staged keys.  Self: key j is visible to row i iff both lie in
        // one trajectory and (causal) j <= i.  Every row sees at least one key (its own position / condition key 0).
        int lo_key[2], hi_key[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qi = r0 + 8 * r;
          if (kSelf) {
            lo_key[r] = qi / args.T * args.T;
            hi_key[r] = args.causal ? qi : lo_key[r] + args.T - 1;
          } else {
            lo_key[r] = 0, hi_key[r] = args.mtok - 1;
          }
        }
        float o[6][4], inv0, inv1;
        attn_hd48_16rows<4>(qf, sK, sV, kKvRow, lo_key, hi_key, sl2, lane, o, inv0, inv1);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          const int col = h * HD + i * 8 + quad * 2;
          *reinterpret_cast<uint32_t*>(sO + sw128_offset(r0, col)) = pack_bf16(o[i][0] * inv0, o[i][1] * inv0);
          *reinterpret_cast<uint32_t*>(sO + sw128_offset(r0 + 8, col)) = pack_bf16(o[i][2] * inv1, o[i][3] * inv1);
        }
      }
      fence_proxy_async_smem();
      consumer_barrier();  // the O tile holds all 8 heads
      // ---- output projection: y[:, 192 g ..] = O · W_o[192 g ..]^T, K = 384
      float y[96] = {};
      mma_k384(y, sO, sW, full, empty, ring, kSlotBytes, g * (kSlotBytes / 2), lane, [] {});
      // ---- epilogue: x = y + b_o + x
      residual_epilogue_192<false>(y, args.x, args.ldx, args.x, args.ldx, args.b_o, row0, nrows, g, r0, quad);
    }
  }
}

template <bool kSelf>
void launch_dec_attn(const bf16* w_in, const bf16* w_o, const DecAttnArgs& a, long rows, cudaStream_t stream) {
  static std::once_flag once;
  std::call_once(once, [] { cudaFuncSetAttribute(dec_attn_kernel<kSelf>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem); });
  const CUtensorMap tmIn = tma_map_2d(w_in, kSelf ? 3 * D : D, D, D, HD, 64, true);
  const CUtensorMap tmO = tma_map_2d(w_o, D, D, D, 192, 64, true);
  const int sms = device_sm_count();
  const int grid = a.tiles < sms ? a.tiles : sms;
  const int N = kSelf ? 4 * D : 2 * D;  // projection output columns: qkv + out, or q + out
  const double flops = 2.0 * rows * (double)N * D;
  const int ticket = prof_begin(flops, (int)rows, N, D, stream);
  dec_attn_kernel<kSelf><<<grid, kThreads, kSmem, stream>>>(tmIn, tmO, a);
  prof_end(ticket, stream);
  prof_count_gemm(flops);
  N1_CUDA(cudaGetLastError());
}

DecAttnArgs dec_args(bf16* x, int ldx, const float* ln_w, const float* ln_b, float eps, const float* b_in, const float* b_o,
                     int B, int Ns, int T) {
  N1_CHECK(x && ln_w && ln_b && b_in && b_o, "dec_attn_block: null pointer");
  N1_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0 && ldx % 8 == 0 && ldx >= D, "dec_attn_block: misaligned x");
  N1_CHECK(B >= 1 && Ns >= 1 && T >= 1 && T <= BM, "dec_attn_block: needs B, Ns >= 1 and 1 <= T <= 64");
  DecAttnArgs a = {};
  a.x = x, a.ldx = ldx, a.ln_w = ln_w, a.ln_b = ln_b, a.eps = eps, a.b_in = b_in, a.b_o = b_o;
  a.Ns = Ns, a.T = T, a.tpt = BM / T;
  a.tiles_per_env = (Ns + a.tpt - 1) / a.tpt;
  const long tiles = (long)B * a.tiles_per_env;
  N1_CHECK(tiles < (1L << 31), "dec_attn_block: too many tiles");
  a.tiles = (int)tiles;
  return a;
}

}  // namespace

void dec_sa_block(bf16* x, int ldx, const float* ln_w, const float* ln_b, float eps, const bf16* w_qkv, const float* b_qkv,
                  const bf16* w_o, const float* b_o, int B, int Ns, int T, int causal, cudaStream_t stream) {
  N1_CHECK(w_qkv && w_o, "dec_sa_block: null weights");
  DecAttnArgs a = dec_args(x, ldx, ln_w, ln_b, eps, b_qkv, b_o, B, Ns, T);
  a.causal = causal ? 1 : 0;
  launch_dec_attn<true>(w_qkv, w_o, a, (long)B * Ns * T, stream);
}

void dec_ca_block(bf16* x, int ldx, const float* ln_w, const float* ln_b, float eps, const bf16* w_q, const float* b_q,
                  const bf16* w_o, const float* b_o, const bf16* kv, int ldkv, int mtok, int B, int Ns, int T,
                  cudaStream_t stream) {
  N1_CHECK(w_q && w_o && kv, "dec_ca_block: null weights or K / V");
  N1_CHECK(mtok >= 1 && mtok <= BM, "dec_ca_block: needs 1 <= condition tokens <= 64");
  N1_CHECK((reinterpret_cast<uintptr_t>(kv) & 15) == 0 && ldkv % 8 == 0 && ldkv >= 2 * D, "dec_ca_block: misaligned K / V");
  DecAttnArgs a = dec_args(x, ldx, ln_w, ln_b, eps, b_q, b_o, B, Ns, T);
  a.kv = kv, a.ldkv = ldkv, a.mtok = mtok;
  launch_dec_attn<false>(w_q, w_o, a, (long)B * Ns * T, stream);
}

}  // namespace n1
