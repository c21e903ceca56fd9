// Persistent warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] @ W[N,K]^T).
//
//   warpgroups 0-1  consumers: each owns 64 of the tile's 128 rows: wgmma m64nBNk16 from shared memory into fp32
//                   register accumulators (one k-block in flight while the previous one's slot is released), then the
//                   epilogue straight from the accumulator fragments: bias / activation / layer-scale / residual, bf16
//                   tiles through a per-warp staging buffer and TMA stores (or direct stores for fp32 / remapped rows).
//   warpgroup 2     producer: one thread of warp 8 issues the TMA loads (cp.async.bulk.tensor 2-D, 128-byte swizzle)
//                   into a STAGES-deep mbarrier ring; warps 9-11 only hand their registers over and leave.
// Tiles are 128 x 256, 128 x 128 or 128 x 64.  384 threads put three warps on every scheduler, so the kernel is compiled
// for 168 registers per thread; after the barrier set-up the producer warpgroup shrinks to 40 and the consumers grow to
// 232 (setmaxnreg), which holds the 128 accumulators of the 256-wide tile plus the epilogue without spilling.
//
// This kernel, one instance per tile width and epilogue kind, carries every Linear / Conv-as-GEMM on the InternVLA-N1 hot
// path (SURVEY.md §2.1):
// the reference reaches cuBLAS through nn.Linear at navdp.py L57-66/L94-100, navdp_backbone.py L147-149,
// dinov2_layers/{attention.py L46-48, mlp.py L30-32, patch_embed.py L65} and the Qwen2.5-VL blocks.
#include <stdlib.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "n1_ops.h"
#include "n1_ptx.cuh"

namespace n1 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 128;  // + the producer warpgroup

template <int BN>
struct Cfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = BN == 256 ? 4 : BN == 128 ? 6 : 8;
  static constexpr int kBarBytes = 256;
  static constexpr int kStoreBytes = kConsumerWarps * 2 * 1024;  // per-warp double-buffered 16x32 bf16 staging for TMA stores
  static constexpr int kSmemBytes = kStages * kStageBytes + kStoreBytes + kBarBytes + 1024;  // +1024: manual alignment
};
static_assert(Cfg<256>::kSmemBytes <= 232448 && Cfg<128>::kSmemBytes <= 232448 && Cfg<64>::kSmemBytes <= 232448,
              "GEMM shared memory budget (227 KB per block)");

constexpr long kWStreamsBytes = 32L << 20;  // a W larger than this streams through the 50 MB L2 instead of living in it

struct GemmArgs {
  int M, N, K;
  int tiles_m, tiles_n;
  void* out;
  int ldo;
  const float* bias;
  const float* gamma;
  const bf16* residual;
  int ldr;
  int act;
  int out_fp32;
  int rows_per_group, group_stride, group_offset;
  const float* row_add;
  int raster_g;  // M tiles per raster group (decode_tile)
};

// Grouped rasterisation: consecutive tile ids walk G M-tiles before moving to the next N-tile, so the CTAs resident at
// one time share few W panels, and the A panels of a group stay L2-resident while the group sweeps all N tiles.  DRAM
// traffic ~ W bytes x (tiles_m / G) + A bytes, so G grows until the group's A panels fill the L2 share given to them.
__device__ __forceinline__ void decode_tile(int tile, int tiles_m, int tiles_n, int G, int& tm, int& tn) {
  const int per_group = G * tiles_n;
  const int g = tile / per_group;
  const int first_m = g * G;
  const int gsize = min(G, tiles_m - first_m);
  const int r = tile - g * per_group;
  tm = first_m + r % gsize;
  tn = r / gsize;
}

// Epilogue kinds.  Each kind is its own compile-time instance of the epilogue below, so an unrolled accumulator loop only
// carries the code of the kind it runs: a tile's epilogue walks a few KB of machine code instead of every activation,
// store path and option inlined at each of its BN / 2 accumulator positions.
//   KIND_LINEAR_SWIGLU  gemm_kernel<BN>: bf16 TMA-store output, acc + bias, then either layer-scale + residual (act none:
//                       every System-2 GEMM but gate/up and the merger's first layer) or SwiGLU (gate/up), picked once
//                       per tile
//   ACT_GELU, ACT_RELU, ACT_GELU_TANH, ACT_SILU   gemm_act_kernel<BN, act>: the same bf16 TMA-store output with one
//                       activation
//   KIND_GENERAL        gemm_act_kernel<BN, KIND_GENERAL>: fp32 output, the output row remap, row_add and outputs no
//                       tensor map can describe, with direct stores; the activation is picked once per tile
constexpr int KIND_LINEAR_SWIGLU = ACT_NONE;
constexpr int KIND_GENERAL = 8;

template <int ACT>
__device__ __forceinline__ float apply_act(float v) {
  if constexpr (ACT == ACT_GELU) return gelu_erf(v);
  else if constexpr (ACT == ACT_RELU) return fmaxf(v, 0.0f);
  else if constexpr (ACT == ACT_GELU_TANH)  // nn.GELU(approximate="tanh"): the NextDiT condition projections
    return 0.5f * v * (1.0f + tanhf(0.7978845608028654f * (v + 0.044715f * v * v * v)));
  else if constexpr (ACT == ACT_SILU) return silu(v);
  else return v;
}

// Epilogue of one tile from the accumulator fragments, for one activation ACT and one store path.  Per element:
// acc + bias -> activation -> layer-scale -> row_add -> residual -> bf16 / fp32 (SwiGLU: (acc + bias) of a (gate, up)
// column pair -> silu(gate) * up).  TMA: the bf16 tile leaves through the warp's staging buffer and bulk tensor stores;
// otherwise direct stores (fp32, the row remap, row_add).
template <int BN, int ACT, bool TMA>
__device__ __forceinline__ void epilogue(const float (&acc)[BN / 2], const GemmArgs& args, const CUtensorMap* tmC, int tm,
                                         int tn, int wrow, int lane, uint8_t* my_store, int& sbuf) {
  constexpr bool kSwiglu = ACT == ACT_SWIGLU;
  const int quad = lane & 3;
  // this thread holds rows r[0], r[1] = r[0] + 8 and, per 8-column group, 2 adjacent columns
  int row[2];
  long out_row[2];
  int grp_row[2] = {0, 0};
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = tm * BM + wrow + (lane >> 2) + h * 8;
    row_ok[h] = row[h] < args.M;
    out_row[h] = row[h];
    if (!TMA && args.rows_per_group > 0) {
      grp_row[h] = row[h] % args.rows_per_group;
      out_row[h] = (long)(row[h] / args.rows_per_group) * args.group_stride + grp_row[h] + args.group_offset;
    }
  }
#pragma unroll
  for (int chunk = 0; chunk < BN / 32; ++chunk) {  // unrolled: the accumulator is indexed statically
    const int col0 = tn * BN + chunk * 32;
    if (col0 >= args.N) break;  // block-uniform
    float v[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = col0 + j * 8 + quad * 2;
      const bool col_ok = col < args.N;
#pragma unroll
      for (int e = 0; e < 4; ++e) v[j][e] = acc[(chunk * 4 + j) * 4 + e];
      if (args.bias && col_ok) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(args.bias + col));
        v[j][0] += b.x, v[j][1] += b.y, v[j][2] += b.x, v[j][3] += b.y;
      }
      if constexpr (kSwiglu) {  // (gate, up) interleaved: this thread's column pair -> one output
        v[j][0] = silu(v[j][0]) * v[j][1];
        v[j][2] = silu(v[j][2]) * v[j][3];
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) v[j][e] = apply_act<ACT>(v[j][e]);
        if (args.gamma && col_ok) {
          const float2 g = __ldg(reinterpret_cast<const float2*>(args.gamma + col));
          v[j][0] *= g.x, v[j][1] *= g.y, v[j][2] *= g.x, v[j][3] *= g.y;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h] || !col_ok) continue;
          if (!TMA && args.row_add) {
            const float2 a = __ldg(reinterpret_cast<const float2*>(args.row_add + (long)grp_row[h] * args.N + col));
            v[j][2 * h] += a.x, v[j][2 * h + 1] += a.y;
          }
          if (args.residual) {
            const uint32_t q = __ldg(reinterpret_cast<const uint32_t*>(args.residual + out_row[h] * args.ldr + col));
            v[j][2 * h] += bf16_lo(q), v[j][2 * h + 1] += bf16_hi(q);
          }
        }
      }
    }
    if constexpr (TMA) {
      // 16 rows x 32 columns (SwiGLU: 16 output columns) staged per warp, then one bulk tensor store.  The staging
      // buffer is 1024-byte aligned and in the tensor map's swizzled layout, which XORs the 16-byte chunk index of a
      // row with the row's address bits 7 and up: 64-byte rows (SWIZZLE_64B) chunk ^= (r >> 1) & 3, 32-byte rows
      // (SWIZZLE_32B) chunk ^= (r >> 2) & 1.  One warp's store then hits every bank once: 4-byte words
      // 16 r + 4 (j ^ (r >> 1) & 3) + quad over r = 0..7, quad = 0..3 are 32 distinct banks (unswizzled: 4-way
      // conflict); SwiGLU's 2-byte stores, 8 r + 4 ((j >> 1) ^ (r >> 2) & 1) + 2 (j & 1) + quad / 2, are 16 distinct
      // banks with two lanes per word (unswizzled: 2-way).
      if (lane == 0) tma_store_wait_read<1>();
      __syncwarp();
      uint8_t* sb = my_store + sbuf * 1024;
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = (lane >> 2) + h * 8;
          if constexpr (kSwiglu)
            *reinterpret_cast<bf16*>(sb + r * 32 + ((((j >> 1) ^ (r >> 2)) & 1) << 4) + (j & 1) * 8 + quad * 2) =
                __float2bfloat16_rn(v[j][2 * h]);
          else
            *reinterpret_cast<uint32_t*>(sb + r * 64 + (((j ^ (r >> 1)) & 3) << 4) + quad * 4) =
                pack_bf16(v[j][2 * h], v[j][2 * h + 1]);
        }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        // rows >= M / cols >= N are clipped by the tensor map
        tma_store_2d(tmC, sb, kSwiglu ? col0 >> 1 : col0, tm * BM + wrow);
        tma_store_commit();
      }
      sbuf ^= 1;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = col0 + j * 8 + quad * 2;
        if (col >= args.N) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h]) continue;
          if constexpr (kSwiglu)
            reinterpret_cast<bf16*>(args.out)[out_row[h] * args.ldo + (col >> 1)] = __float2bfloat16_rn(v[j][2 * h]);
          else if (args.out_fp32)
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(args.out) + out_row[h] * args.ldo + col) =
                make_float2(v[j][2 * h], v[j][2 * h + 1]);
          else
            *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(args.out) + out_row[h] * args.ldo + col) =
                pack_bf16(v[j][2 * h], v[j][2 * h + 1]);
        }
      }
    }
  }
}

// The persistent kernel with the epilogue of KIND (above); every kind but KIND_GENERAL stores through TMA.
template <int BN, int KIND>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                                          const GemmArgs& args) {
  using C = Cfg<BN>;
  constexpr bool kTma = KIND != KIND_GENERAL;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + C::kStages * C::kABytes;
  uint8_t* sStore = smem + C::kStages * C::kStageBytes;  // 1024-byte aligned: the swizzled staging layout needs it
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStore + C::kStoreBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + C::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = args.tiles_m * args.tiles_n;
  const int nkb = (args.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (kTma) tma_prefetch_desc(&tmC);
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumerWarps);  // every consumer warp releases the slot once its own MMAs have read it
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int tm, tn;
        decode_tile(tile, args.tiles_m, args.tiles_n, args.raster_g, tm, tn);
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], C::kStageBytes);
          tma_load_2d(sA + stage * C::kABytes, &tmA, &full[stage], kb * BK, tm * BM);
          tma_load_2d(sB + stage * C::kBBytes, &tmB, &full[stage], kb * BK, tn * BN);
          if (++stage == C::kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: main loop + epilogue
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2;               // consumer warpgroup: rows [64 wg, 64 wg + 64) of the tile
    const int wrow = wg * 64 + (warp & 3) * 16;  // first of this warp's 16 rows
    uint8_t* my_store = sStore + warp * 2048;
    int sbuf = 0;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int tm, tn;
      decode_tile(tile, args.tiles_m, args.tiles_n, args.raster_g, tm, tn);
      float acc[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = wgmma_desc_sw128(smem_u32(sA + stage * C::kABytes + wg * 64 * 128));
        const uint64_t bdesc = wgmma_desc_sw128(smem_u32(sB + stage * C::kBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)  // 16 elements (32 bytes) along K inside the swizzle row: +2 in 16-byte units
          wgmma_ss<0, 0>(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have read their slot
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == C::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      // ---- epilogue: one compile-time kind per branch, chosen once per tile (block-uniform)
#define N1_EPI(act, tma) epilogue<BN, act, tma>(acc, args, &tmC, tm, tn, wrow, lane, my_store, sbuf)
      if constexpr (KIND == KIND_LINEAR_SWIGLU) {
        if (args.act == ACT_SWIGLU) N1_EPI(ACT_SWIGLU, true);
        else N1_EPI(ACT_NONE, true);
      } else if constexpr (KIND == KIND_GENERAL) {
        switch (args.act) {
          case ACT_GELU: N1_EPI(ACT_GELU, false); break;
          case ACT_RELU: N1_EPI(ACT_RELU, false); break;
          case ACT_SWIGLU: N1_EPI(ACT_SWIGLU, false); break;
          case ACT_GELU_TANH: N1_EPI(ACT_GELU_TANH, false); break;
          case ACT_SILU: N1_EPI(ACT_SILU, false); break;
          default: N1_EPI(ACT_NONE, false); break;
        }
      } else {
        N1_EPI(KIND, true);
      }
#undef N1_EPI
    }
    if (kTma && lane == 0) tma_store_wait<0>();
    __syncwarp();
  }
}

// The linear and SwiGLU kinds: every System-2 GEMM but the merger's first layer.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC, const GemmArgs args) {
  gemm_body<BN, KIND_LINEAR_SWIGLU>(tmA, tmB, tmC, args);
}

// One activation per instance (KIND = ACT_GELU / ACT_RELU / ACT_GELU_TANH / ACT_SILU), or KIND_GENERAL.
template <int BN, int KIND>
__global__ void __launch_bounds__(kThreads, 1)
gemm_act_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmC, const GemmArgs args) {
  gemm_body<BN, KIND>(tmA, tmB, tmC, args);
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  if (!fn) throw Error(-4, "cuTensorMapEncodeTiled unavailable (no CUDA driver / GPU?)");
  return fn;
}

// 2-D bf16 tensor map over a row-major [rows, cols] matrix with leading dimension ld; box = [box_rows, box_cols];
// operands use box_cols = 64 with the 128-byte swizzle, output staging tiles the 64-byte (32 columns) or 32-byte
// (SwiGLU's 16 columns) one.
CUtensorMap make_map(const bf16* ptr, long rows, long cols, long ld, int box_rows, int box_cols = BK,
                     CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  N1_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "GEMM operand not 16-byte aligned");
  N1_CHECK(ld % 8 == 0, "GEMM operand leading dimension must be a multiple of 8 elements");
  CUtensorMap m;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16*>(ptr), gdim, gstr, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(-5, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  return m;
}

template <int BN, int KIND>
constexpr auto kernel_of() {
  if constexpr (KIND == KIND_LINEAR_SWIGLU) return gemm_kernel<BN>;
  else return gemm_act_kernel<BN, KIND>;
}

template <int BN, int KIND>
void launch(const bf16* A, int lda, const bf16* W, int ldw, int M, int N, int K, GemmArgs& a, cudaStream_t stream) {
  using C = Cfg<BN>;
  auto* kernel = kernel_of<BN, KIND>();
  static std::once_flag once;
  std::call_once(once, [kernel] {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
  });
  a.tiles_m = (M + BM - 1) / BM;
  a.tiles_n = (N + BN - 1) / BN;
  {
    // raster group: as many M tiles of A as fit a third of the 50 MB L2 (W streams through the rest); only matters
    // when W does not fit L2.  The SMs hold sms / G W panels at a time: at K = 3584 (G = 18) that is 7 panels, 6.4 MB
    // with the 128-wide tile and 12.8 MB with the 256-wide one, which still leaves the rest of the L2 to the stream,
    // so G does not depend on BN.
    const long panel = (long)BM * K * 2;
    const long w_bytes = (long)N * K * 2;
    int g = 8;
    if (w_bytes > kWStreamsBytes) g = (int)std::max<long>(2, (16L << 20) / panel);
    a.raster_g = g < a.tiles_m ? g : a.tiles_m;
    if (a.raster_g < 1) a.raster_g = 1;
  }
  CUtensorMap tmA = make_map(A, M, K, lda, BM);
  CUtensorMap tmB = make_map(W, N, K, ldw, BN);
  CUtensorMap tmC = tmA;  // placeholder for the direct-store epilogue (KIND_GENERAL)
  if (KIND != KIND_GENERAL) {
    const bool sw = a.act == ACT_SWIGLU;
    tmC = make_map(static_cast<const bf16*>(a.out), M, sw ? N / 2 : N, a.ldo, 16, sw ? 16 : 32,
                   sw ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_64B);
  }
  const int tiles = a.tiles_m * a.tiles_n;
  const int grid = tiles < device_sm_count() ? tiles : device_sm_count();
  kernel<<<grid, kThreads, C::kSmemBytes, stream>>>(tmA, tmB, tmC, a);
  N1_CUDA(cudaGetLastError());
}

template <int BN>
void launch_kind(int kind, const bf16* A, int lda, const bf16* W, int ldw, int M, int N, int K, GemmArgs& a,
                 cudaStream_t stream) {
  switch (kind) {
    case KIND_LINEAR_SWIGLU: return launch<BN, KIND_LINEAR_SWIGLU>(A, lda, W, ldw, M, N, K, a, stream);
    case ACT_GELU: return launch<BN, ACT_GELU>(A, lda, W, ldw, M, N, K, a, stream);
    case ACT_RELU: return launch<BN, ACT_RELU>(A, lda, W, ldw, M, N, K, a, stream);
    case ACT_GELU_TANH: return launch<BN, ACT_GELU_TANH>(A, lda, W, ldw, M, N, K, a, stream);
    case ACT_SILU: return launch<BN, ACT_SILU>(A, lda, W, ldw, M, N, K, a, stream);
    default: return launch<BN, KIND_GENERAL>(A, lda, W, ldw, M, N, K, a, stream);
  }
}

// ---- profiling state
std::atomic<long> g_total_launches{0}, g_gemm_launches{0};
std::atomic<bool> g_prof_on{false};
std::mutex g_prof_mu;
struct EvPair {
  cudaEvent_t a, b;
  double flops;
  int M, N, K;
};
std::vector<EvPair> g_events;
struct ShapeAcc {
  int M, N, K;
  long count;
  double ms;
};
std::vector<ShapeAcc> g_shapes;  // per-(M, N, K) sums of the event-timed launches since the last prof_read_shapes()

}  // namespace

CUtensorMap tma_map_2d(const bf16* ptr, long rows, long cols, long ld, int box_rows, int box_cols, bool swizzle) {
  return make_map(ptr, rows, cols, ld, box_rows, box_cols, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE);
}
CUtensorMap tma_map_3d_sw128(const bf16* ptr, const long dims[3], const long strides[2], const int box[3]) {
  N1_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && strides[0] % 8 == 0 && strides[1] % 8 == 0,
           "tma_map_3d_sw128: 16-byte alignment");
  CUtensorMap m;
  cuuint64_t gdim[3] = {(cuuint64_t)dims[0], (cuuint64_t)dims[1], (cuuint64_t)dims[2]};
  cuuint64_t gstr[2] = {(cuuint64_t)strides[0] * 2, (cuuint64_t)strides[1] * 2};
  cuuint32_t bx[3] = {(cuuint32_t)box[0], (cuuint32_t)box[1], (cuuint32_t)box[2]};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<bf16*>(ptr), gdim, gstr, bx, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(-5, "cuTensorMapEncodeTiled (3-D) failed: " + std::to_string((int)r));
  return m;
}
// Counts one GEMM-class launch: gemm_bf16 and the fused decoder kernels in other files
void prof_count_gemm(double flops) {
  (void)flops;
  g_gemm_launches++;
  g_total_launches++;
}

void prof_enable(bool on) { g_prof_on = on; }
// Event bracket of a GEMM-class launch (gemm_bf16 and the fused decoder blocks): returns a ticket (< 0: off)
int prof_begin(double flops, int M, int N, int K, cudaStream_t s) {
  if (!g_prof_on.load()) return -1;
  EvPair ev{};
  cudaEventCreate(&ev.a);
  cudaEventCreate(&ev.b);
  ev.flops = flops, ev.M = M, ev.N = N, ev.K = K;
  cudaEventRecord(ev.a, s);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_events.push_back(ev);
  return (int)g_events.size() - 1;
}
void prof_end(int ticket, cudaStream_t s) {
  if (ticket < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (ticket < (int)g_events.size()) cudaEventRecord(g_events[ticket].b, s);
}
void prof_count_launch(int n) { g_total_launches += n; }
ProfStats prof_read_and_reset() {
  ProfStats st;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (EvPair& e : g_events) {
    cudaEventSynchronize(e.b);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e.a, e.b) == cudaSuccess) {
      st.gemm_ms += ms, st.gemm_flops += e.flops;
      bool hit = false;
      for (ShapeAcc& sa : g_shapes)
        if (sa.M == e.M && sa.N == e.N && sa.K == e.K) {
          sa.count++, sa.ms += ms, hit = true;
          break;
        }
      if (!hit) g_shapes.push_back({e.M, e.N, e.K, 1, (double)ms});
    }
    cudaEventDestroy(e.a);
    cudaEventDestroy(e.b);
  }
  g_events.clear();
  st.gemm_launches = g_gemm_launches.exchange(0);
  st.total_launches = g_total_launches.exchange(0);
  return st;
}

int prof_read_shapes(int* mnk, long* count, double* ms, int cap) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  int n = 0;
  for (const ShapeAcc& sa : g_shapes) {
    if (n >= cap) break;
    mnk[3 * n] = sa.M, mnk[3 * n + 1] = sa.N, mnk[3 * n + 2] = sa.K;
    count[n] = sa.count, ms[n] = sa.ms;
    ++n;
  }
  g_shapes.clear();
  return n;
}

int device_sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

void gemm_bf16(const bf16* A, int lda, const bf16* W, int ldw, void* out, int ldo, int M, int N, int K,
               const GemmEpilogue& e, cudaStream_t stream, int tile_n) {
  if (M <= 0 || N <= 0) return;
  N1_CHECK(tile_n == 0 || tile_n == 64 || tile_n == 128 || tile_n == 256, "GEMM tile width must be 0, 64, 128 or 256");
  N1_CHECK(K > 0 && K % 8 == 0, "GEMM K must be a positive multiple of 8");
  N1_CHECK(N % 8 == 0, "GEMM N must be a multiple of 8 (pad the packed weight)");
  N1_CHECK(!(e.act == ACT_SWIGLU) || N % 16 == 0, "SwiGLU GEMM needs N % 16 == 0");
  GemmArgs a;
  a.M = M, a.N = N, a.K = K;
  a.out = out, a.ldo = ldo;
  a.bias = e.bias, a.gamma = e.gamma, a.residual = e.residual, a.ldr = e.ldr;
  a.act = e.act, a.out_fp32 = e.out_fp32;
  a.rows_per_group = e.rows_per_group, a.group_stride = e.group_stride, a.group_offset = e.group_offset;
  a.row_add = e.row_add;
  // bf16 output tiles leave through smem staging and TMA stores (full-sector writes) wherever a tensor map can describe
  // the output; the activation then picks the kernel instance, and everything else takes the general direct-store path
  const bool tma = !e.out_fp32 && e.rows_per_group == 0 && !e.row_add && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                   ldo % 8 == 0;
  int kind = KIND_GENERAL;
  if (tma) {
    kind = KIND_LINEAR_SWIGLU;  // also an act value outside GemmAct, which the epilogue has always treated as none
    if (e.act == ACT_GELU || e.act == ACT_RELU || e.act == ACT_GELU_TANH || e.act == ACT_SILU) kind = e.act;
  }
  // Tile-width choice from the shape and the SM count: the least waves x (BN + fixed prologue / epilogue share), ties to
  // the wider tile (fewer A re-reads, longer MMA bursts).  The 256-wide tile is a candidate only when W does not fit the
  // L2 (the raster rule's test in launch()): there the 128-wide tile is held back by operand traffic and 256 wins (LLM
  // gate/up and down projections, DESIGN.md §5); where W is L2-resident its longer epilogue, during which the tensor
  // cores idle, costs more than it saves.  tile_n != 0 (tests and scripts/bench_tiles.py) overrides the choice.
  const int sms = device_sm_count();
  const int tm = (M + BM - 1) / BM;
  auto cost = [&](int bn) {
    const long tiles = (long)tm * ((N + bn - 1) / bn);
    const long waves = (tiles + sms - 1) / sms;
    return waves * (bn + 48);
  };
  int bn = tile_n;
  if (bn == 0) {
    bn = cost(128) <= cost(64) ? 128 : 64;
    if ((long)N * K * 2 > kWStreamsBytes && cost(256) <= cost(bn)) bn = 256;
  }
  const double flops = 2.0 * M * (double)N * K;
  const int ticket = prof_begin(flops, M, N, K, stream);
  prof_count_gemm(flops);
  if (bn == 256) launch_kind<256>(kind, A, lda, W, ldw, M, N, K, a, stream);
  else if (bn == 128) launch_kind<128>(kind, A, lda, W, ldw, M, N, K, a, stream);
  else launch_kind<64>(kind, A, lda, W, ldw, M, N, K, a, stream);
  prof_end(ticket, stream);
}

}  // namespace n1
