// Tile code shared by the fused NavDP decoder kernels (ff_block.cu, dec_attn_block.cu) and the short-sequence attention
// kernel (attention.cu).  The fused kernels work on 64-row tiles of the D = 384 residual stream: two consumer warpgroups,
// warp cw (0..7) of them owning rows 8 cw .. 8 cw + 7 of the LayerNorm prologue and rows (cw % 4) * 16 + lane / 4 (+ 8) of
// every wgmma accumulator; operands live in shared memory as K-major tiles of 64-column k-blocks with the 128-byte swizzle.
#pragma once
#include "n1_ops.h"
#include "n1_ptx.cuh"

namespace n1 {

// Byte offset of bf16 element (row, col) in a K-major tile of 64-row, 64-column k-blocks (8192 bytes each) with the
// 128-byte swizzle: k-block col / 64, 8-row group row / 8, 16-byte chunk (col % 64) / 8 stored at position chunk ^ (row % 8).
__device__ __forceinline__ int sw128_offset(int row, int col) {
  return (col >> 6) * 8192 + (row >> 3) * 1024 + (row & 7) * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
}

// Slot and phase of an mbarrier ring of kS slots.
template <int kS>
struct Ring {
  int slot = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++slot == kS) slot = 0, phase ^= 1;
  }
};

// LayerNorm of rows row0 .. row0 + 63 of x (384 bf16 columns) into the bf16 A tile sA (6 swizzled k-blocks, 48 KB); rows
// at or past nrows read as zeros.  Warp cw normalises rows 8 cw .. 8 cw + 7 with coalesced 8-byte loads and a two-pass
// variance; all 24 loads of its 8 rows are issued before the first use and the shuffle reductions advance in lock-step.
// kNc: read x through the non-coherent path (x is not written by this kernel before the read).
template <bool kNc>
__device__ __forceinline__ void ln384_to_tile(uint8_t* sA, const bf16* x, long ldx, long row0, int nrows, const float* ln_w,
                                              const float* ln_b, float eps, int cw, int lane) {
  constexpr int D = 384;
  uint2 q[8][3];
#pragma unroll
  for (int rr = 0; rr < 8; ++rr) {
    const int r = cw * 8 + rr;
    const uint2* xr = reinterpret_cast<const uint2*>(x + (row0 + r) * ldx);
#pragma unroll
    for (int i = 0; i < 3; ++i)
      q[rr][i] = r < nrows ? (kNc ? __ldg(xr + lane + i * 32) : xr[lane + i * 32]) : make_uint2(0u, 0u);
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
    const float4 lw = __ldg(reinterpret_cast<const float4*>(ln_w + col));
    const float4 lb = __ldg(reinterpret_cast<const float4*>(ln_b + col));
#pragma unroll
    for (int rr = 0; rr < 8; ++rr) {
      const float mu = s[rr], rstd = rsqrtf(sq[rr] * (1.0f / D) + eps);
      const float y0 = (bf16_lo(q[rr][i].x) - mu) * rstd * lw.x + lb.x, y1 = (bf16_hi(q[rr][i].x) - mu) * rstd * lw.y + lb.y;
      const float y2 = (bf16_lo(q[rr][i].y) - mu) * rstd * lw.z + lb.z, y3 = (bf16_hi(q[rr][i].y) - mu) * rstd * lw.w + lb.w;
      *reinterpret_cast<uint2*>(sA + sw128_offset(cw * 8 + rr, col)) = make_uint2(pack_bf16(y0, y1), pack_bf16(y2, y3));
    }
  }
}

// acc[64 x N] = A · B^T with K = 384: A the swizzled tile sA, B one k-block per slot of the weight ring (full / empty
// mbarriers, slot s at ring + s * slot_bytes, this warpgroup's rows b_offset bytes into it).  Six k-blocks of 4 wgmma
// k-steps; each k-block's slot is released (by lane 0 of every consumer warp) once the next k-block's MMAs are issued
// and the earlier ones complete.  after_first() runs right after the first wgmma_wait<1>, when every MMA group committed
// before this call has completed.
template <int N, int kS, typename AfterFirst>
__device__ __forceinline__ void mma_k384(float (&acc)[N], const uint8_t* sA, const uint8_t* ring, uint64_t* full,
                                         uint64_t* empty, Ring<kS>& rs, int slot_bytes, int b_offset, int lane,
                                         AfterFirst after_first) {
  int prev = -1;
#pragma unroll 1
  for (int kb = 0; kb < 6; ++kb) {
    mbar_wait(&full[rs.slot], rs.phase);
    const uint64_t ad = wgmma_desc_sw128(smem_u32(sA + kb * 8192));
    const uint64_t bd = wgmma_desc_sw128(smem_u32(ring + rs.slot * slot_bytes + b_offset));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<0, 0>(acc, ad + 2 * k, bd + 2 * k, (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (kb == 0) after_first();
    if (lane == 0 && prev >= 0) mbar_arrive(&empty[prev]);
    prev = rs.slot;
    rs.advance();
  }
  wgmma_wait<0>();
  if (lane == 0) mbar_arrive(&empty[prev]);
}

// out = y + bias + x as bf16 over the warpgroup's 192 output columns 192 g .. of rows row0 + r0 and row0 + r0 + 8 (those
// below nrows); y is the m64n192k16 accumulator.  A thread re-reads exactly the elements it overwrites, so out may be x.
template <bool kNc>
__device__ __forceinline__ void residual_epilogue_192(const float (&y)[96], const bf16* x, long ldx, bf16* out, long ldo,
                                                      const float* bias, long row0, int nrows, int g, int r0, int quad) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = r0 + hh * 8;
    if (r >= nrows) continue;
    const bf16* xr = x + (row0 + r) * ldx + g * 192 + quad * 2;
    bf16* orow = out + (row0 + r) * ldo + g * 192 + quad * 2;
#pragma unroll
    for (int jj = 0; jj < 24; ++jj) {
      const uint32_t* xp = reinterpret_cast<const uint32_t*>(xr + jj * 8);
      const uint32_t xv = kNc ? __ldg(xp) : *xp;
      const float2 b = __ldg(reinterpret_cast<const float2*>(bias + g * 192 + jj * 8 + quad * 2));
      *reinterpret_cast<uint32_t*>(orow + jj * 8) =
          pack_bf16(y[jj * 4 + 2 * hh] + bf16_lo(xv) + b.x, y[jj * 4 + 2 * hh + 1] + bf16_hi(xv) + b.y);
    }
  }
}

// Attention of one warp's 16 query rows over up to 16 NKP keys, head dim 48, on mma.sync.m16n8k16: S = Q K^T, the masked
// softmax in fp32 (P rounded to bf16), O = P V.  qf: Q as A fragments (3 k-steps of 16).  Key j sits at sK / sV +
// j * row_bytes (48 contiguous bf16).  Row lane / 4 (r = 0) and row lane / 4 + 8 (r = 1) see key j iff
// lo_key[r] <= j <= hi_key[r]; a row that sees no key gets O = 0.  Returns the unnormalised O (o[i]: columns 8 i ..) and
// the reciprocal row sums inv0 / inv1.
template <int NKP>
__device__ __forceinline__ void attn_hd48_16rows(const uint32_t (&qf)[3][4], const uint8_t* sK, const uint8_t* sV,
                                                 int row_bytes, const int (&lo_key)[2], const int (&hi_key)[2], float sl2,
                                                 int lane, float (&o)[6][4], float& inv0, float& inv1) {
  const int lm = lane >> 3, lr = lane & 7;  // ldmatrix: matrix / row of this lane's address
  float s[2 * NKP][4];
#pragma unroll
  for (int i = 0; i < 2 * NKP; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 3; ++ks)
#pragma unroll
    for (int np = 0; np < NKP; ++np) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4(smem_u32(sK + (np * 16 + (lm >> 1) * 8 + lr) * row_bytes + (ks * 16 + (lm & 1) * 8) * 2), b0, b1, b2, b3);
      mma_bf16(s[2 * np], qf[ks], b0, b1);
      mma_bf16(s[2 * np + 1], qf[ks], b2, b3);
    }
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 2 * NKP; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int key = i * 8 + (lane & 3) * 2 + (e & 1), r = e >> 1;
      const bool vis = key >= lo_key[r] && key <= hi_key[r];
      s[i][e] = vis ? s[i][e] * sl2 : -INFINITY;
      mx[r] = fmaxf(mx[r], s[i][e]);
    }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    if (mx[r] == -INFINITY) mx[r] = 0.f;
  }
  uint32_t pf[NKP][4];
#pragma unroll
  for (int i = 0; i < 2 * NKP; ++i) {
    const float p0 = exp2f(s[i][0] - mx[0]), p1 = exp2f(s[i][1] - mx[0]);
    const float p2 = exp2f(s[i][2] - mx[1]), p3 = exp2f(s[i][3] - mx[1]);
    sum[0] += p0 + p1, sum[1] += p2 + p3;
    pf[i >> 1][(i & 1) * 2 + 0] = pack_bf16(p0, p1);
    pf[i >> 1][(i & 1) * 2 + 1] = pack_bf16(p2, p3);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < NKP; ++kk)
#pragma unroll
    for (int np = 0; np < 3; ++np) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4_t(smem_u32(sV + (kk * 16 + (lm & 1) * 8 + lr) * row_bytes + (np * 16 + (lm >> 1) * 8) * 2), b0, b1, b2, b3);
      mma_bf16(o[2 * np], pf[kk], b0, b1);
      mma_bf16(o[2 * np + 1], pf[kk], b2, b3);
    }
  inv0 = sum[0] > 0.f ? 1.f / sum[0] : 0.f;
  inv1 = sum[1] > 0.f ? 1.f / sum[1] : 0.f;
}

}  // namespace n1
