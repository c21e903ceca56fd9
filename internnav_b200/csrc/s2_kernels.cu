// Glue kernels of the System-2 path (Qwen2.5-VL ViT + decoder prefill): row gathers, rotary tables and application,
// embedding splice.  Reference arithmetic: transformers==4.51.0 modeling_qwen2_5_vl.py (un-vendored pin,
// requirements/internvla_n1.txt L7) as called from internvla_n1.py L320-347; restated in oracle/qwen_oracle.py.
#include "s2_kernels.h"

#include "n1_ptx.cuh"

namespace n1 {
namespace {

__global__ void gather_rows_kernel(const bf16* __restrict__ src, const int* __restrict__ idx, bf16* __restrict__ dst,
                                   const int* __restrict__ dst_idx, long rows, int group, int vec_per_row) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * vec_per_row) return;
  const long r = i / vec_per_row;
  const int c = i % vec_per_row;
  const long sr = (long)idx[r / group] * group + r % group;
  const long dr = dst_idx ? (long)dst_idx[r / group] * group + r % group : r;
  reinterpret_cast<uint4*>(dst)[dr * vec_per_row + c] = __ldg(reinterpret_cast<const uint4*>(src) + sr * vec_per_row + c);
}

__global__ void vit_rope_table_kernel(const int* __restrict__ pos_hw, float2* __restrict__ cs, long tokens, int half,
                                      float theta) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tokens * half) return;
  const long t = i / half;
  const int j = i % half;
  const int q = half / 2;  // frequencies per axis
  const int p = pos_hw[t * 2 + (j < q ? 0 : 1)];
  // inv_freq = 1 / theta^(arange(0, dim, 2) / dim) with dim = half (Qwen2_5_VisionRotaryEmbedding(head_dim // 2))
  const float inv = 1.0f / powf(theta, (float)(2 * (j % q)) / (float)half);
  float sn, cn;
  sincosf((float)p * inv, &sn, &cn);
  cs[i] = make_float2(cn, sn);
}

__global__ void mrope_table_kernel(const int* __restrict__ pos3, float2* __restrict__ cs, long tokens, int half,
                                   int sec_t, int sec_h, float theta) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tokens * half) return;
  const long t = i / half;
  const int j = i % half;
  const int stream = j < sec_t ? 0 : (j < sec_t + sec_h ? 1 : 2);
  const int p = pos3[(long)stream * tokens + t];
  const float inv = 1.0f / powf(theta, (float)(2 * j) / (float)(2 * half));
  float sn, cn;
  sincosf((float)p * inv, &sn, &cn);
  cs[i] = make_float2(cn, sn);
}

// 8 rotation pairs (two 16-byte vectors) per thread; half % 8 == 0.
__global__ void apply_rope_kernel(bf16* __restrict__ x, int ld, const float2* __restrict__ cs, long tokens, int heads,
                                  int half) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int vec = half / 8;
  const long per_tok = (long)heads * vec;
  if (i >= tokens * per_tok) return;
  const long t = i / per_tok;
  const int h = (i % per_tok) / vec, j = (i % vec) * 8;
  bf16* p = x + t * ld + (long)h * 2 * half + j;
  uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(p + half);
  const float4* c4 = reinterpret_cast<const float4*>(cs + t * half + j);  // (cos, sin) pairs
  uint32_t* au = reinterpret_cast<uint32_t*>(&a);
  uint32_t* bu = reinterpret_cast<uint32_t*>(&b);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 c = __ldg(c4 + k);  // c.x,c.y = cos,sin of pair 2k ; c.z,c.w of pair 2k+1
    const float a0 = bf16_lo(au[k]), a1 = bf16_hi(au[k]), b0 = bf16_lo(bu[k]), b1 = bf16_hi(bu[k]);
    au[k] = pack_bf16(a0 * c.x - b0 * c.y, a1 * c.z - b1 * c.w);
    bu[k] = pack_bf16(b0 * c.x + a0 * c.y, b1 * c.z + a1 * c.w);
  }
  *reinterpret_cast<uint4*>(p) = a;
  *reinterpret_cast<uint4*>(p + half) = b;
}

__global__ void build_embeds_kernel(const int* __restrict__ kind, const int* __restrict__ src,
                                    const bf16* __restrict__ emb, const bf16* __restrict__ img,
                                    const bf16* __restrict__ lat, const int* __restrict__ img_rows,
                                    bf16* __restrict__ out, long tokens, int vec_per_row) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tokens * vec_per_row) return;
  const long t = i / vec_per_row;
  const int c = i % vec_per_row;
  const int k = kind[t];
  const bf16* base = k == 0 ? emb : (k == 1 ? img : lat);
  const long row = k == 1 && img_rows ? img_rows[src[t]] : src[t];
  reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(base) + row * vec_per_row + c);
}


// ---- greedy decode bookkeeping (internvla_n1_policy.py L169-176: model.generate(do_sample=False, max_new_tokens=128))
// Sequence b has `len[b]` prompt tokens and has sampled `gen[b]` tokens so far.  The next chunk holds the tokens with
// in-sequence indices idx = len + gen - back + j, j in [0, per_seq): their cache rows, rotary positions (text tokens
// after the prompt sit at idx + delta on all three mrope axes, rope2d.py L150-160) and the visible key count.
__global__ void gen_rows_kernel(const int* __restrict__ len, const int* __restrict__ delta, const int* __restrict__ gen,
                                int back, int per_seq, int B, int slot, const int* __restrict__ row0,
                                const int* __restrict__ pages, int* __restrict__ dest_rows, int* __restrict__ pos3,
                                int* __restrict__ k_len) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * per_seq) return;
  const int b = i / per_seq, j = i % per_seq;
  const int idx = len[b] + gen[b] - back + j;
  const int r = (row0 ? row0[b] : b * slot) + idx;
  dest_rows[i] = pages ? pages[r >> 6] * 64 + (r & 63) : r;
  const int rows = B * per_seq;
  pos3[i] = pos3[rows + i] = pos3[2 * rows + i] = idx + delta[b];
  if (j == per_seq - 1) k_len[b] = idx + 1;
}

__global__ void page_rows_kernel(const int* __restrict__ rows, const int* __restrict__ pages, int* __restrict__ out,
                                 long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rows[i];
  out[i] = pages[r >> 6] * 64 + (r & 63);
}

// K and V column blocks of the packed qkv rows -> rows dest_rows[r] of the layer's cache ([*, kvdim] each)
__global__ void kv_append_kernel(const bf16* __restrict__ qkv, int ld, int k_off, int v_off, int vec_per_row,
                                 const int* __restrict__ dest_rows, long rows, bf16* __restrict__ ck,
                                 bf16* __restrict__ cv) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * vec_per_row) return;
  const long r = i / vec_per_row;
  const int c = i % vec_per_row;
  const long d = (long)dest_rows[r] * vec_per_row + c;
  reinterpret_cast<uint4*>(ck)[d] = *reinterpret_cast<const uint4*>(qkv + r * ld + k_off + c * 8);
  reinterpret_cast<uint4*>(cv)[d] = *reinterpret_cast<const uint4*>(qkv + r * ld + v_off + c * 8);
}

// rows of the latent pass: [last sampled token, latent_queries[0..nq)] per sequence
__global__ void latent_src_kernel(const int* __restrict__ cur_tok, int B, int nq, int* __restrict__ kind,
                                  int* __restrict__ src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * (nq + 1)) return;
  const int b = i / (nq + 1), j = i % (nq + 1);
  kind[i] = j == 0 ? 0 : 2;
  src[i] = j == 0 ? cur_tok[b] : j - 1;
}

// torch.argmax over bf16 logits: the FIRST index holding the maximum.  One CTA per row.
__global__ void __launch_bounds__(256) argmax_rows_kernel(const bf16* __restrict__ logits, long ld, int n,
                                                          int* __restrict__ out) {
  const bf16* row = logits + (long)blockIdx.x * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n; i += 256) {
    const float v = __bfloat162float(row[i]);
    if (v > best || (v == best && i < bi)) best = v, bi = i;
  }
  __shared__ float sv[256];
  __shared__ int si[256];
  sv[threadIdx.x] = best, si[threadIdx.x] = bi;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if (threadIdx.x < k) {
      const float v = sv[threadIdx.x + k];
      const int j = si[threadIdx.x + k];
      if (v > sv[threadIdx.x] || (v == sv[threadIdx.x] && j < si[threadIdx.x])) sv[threadIdx.x] = v, si[threadIdx.x] = j;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = si[0] == 0x7fffffff ? 0 : si[0];
}

// Accept the sampled token of every unfinished sequence; EOS or the token budget finishes it (GenerationMixin greedy
// search: finished rows are padded, the EOS token itself is part of the output).  *n_active = sequences still running.
__global__ void gen_update_kernel(const int* __restrict__ next, int* __restrict__ cur_tok, int* __restrict__ gen,
                                  int* __restrict__ finished, int* __restrict__ out_tokens, int max_new, int eos0, int eos1,
                                  int eos2, int eos3, int B, int* __restrict__ n_active) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (finished[b]) return;
  const int t = next[b];
  out_tokens[(long)b * max_new + gen[b]] = t;
  cur_tok[b] = t;
  const int g = ++gen[b];
  if (t == eos0 || t == eos1 || t == eos2 || t == eos3 || g >= max_new) finished[b] = 1;
  else atomicAdd(n_active, 1);
}

__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
// one CTA per image; a sum of per-word hashes, so the reduction order does not matter
__global__ void __launch_bounds__(256) image_digest_kernel(const uint32_t* __restrict__ words, long words_per_row,
                                                           const int64_t* __restrict__ row_off, uint64_t* __restrict__ out) {
  const long w0 = row_off[blockIdx.x] * words_per_row, n = (row_off[blockIdx.x + 1] - row_off[blockIdx.x]) * words_per_row;
  uint64_t h = 0;
  for (long j = threadIdx.x; j < n; j += 256) h += splitmix64(((uint64_t)j << 32) | words[w0 + j]);
  for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  __shared__ unsigned long long acc;
  if (threadIdx.x == 0) acc = (unsigned long long)n;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicAdd(&acc, (unsigned long long)h);
  __syncthreads();
  if (threadIdx.x == 0) out[blockIdx.x] = acc;
}

inline int nblk(long n) { return (int)((n + 255) / 256); }

}  // namespace

void gather_rows(const bf16* src, const int* idx, bf16* dst, long rows, int group, int cols, cudaStream_t s,
                 const int* dst_idx) {
  N1_CHECK(cols % 8 == 0, "gather_rows: cols % 8");
  gather_rows_kernel<<<nblk(rows * (cols / 8)), 256, 0, s>>>(src, idx, dst, dst_idx, rows, group, cols / 8);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void vit_rope_table(const int* pos_hw, float2* cs, long tokens, int half, float theta, cudaStream_t s) {
  vit_rope_table_kernel<<<nblk(tokens * half), 256, 0, s>>>(pos_hw, cs, tokens, half, theta);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void mrope_table(const int* pos3, float2* cs, long tokens, int half, int sec_t, int sec_h, float theta,
                 cudaStream_t s) {
  mrope_table_kernel<<<nblk(tokens * half), 256, 0, s>>>(pos3, cs, tokens, half, sec_t, sec_h, theta);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void apply_rope(bf16* x, int ld, const float2* cs, long tokens, int heads, int hd, cudaStream_t s) {
  N1_CHECK((hd / 2) % 8 == 0 && ld % 8 == 0, "apply_rope: head_dim / 2 and ld must be multiples of 8");
  apply_rope_kernel<<<nblk(tokens * heads * (hd / 16)), 256, 0, s>>>(x, ld, cs, tokens, heads, hd / 2);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void build_embeds(const int* kind, const int* src, const bf16* embed_tokens, const bf16* image_feats,
                  const bf16* latent_queries, bf16* out, long tokens, int H, cudaStream_t s, const int* image_rows) {
  N1_CHECK(H % 8 == 0, "build_embeds: H % 8");
  build_embeds_kernel<<<nblk(tokens * (H / 8)), 256, 0, s>>>(kind, src, embed_tokens, image_feats, latent_queries,
                                                            image_rows, out, tokens, H / 8);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

void gen_rows(const int* len, const int* delta, const int* gen, int back, int per_seq, int B, int slot, const int* row0,
              const int* pages, int* dest_rows, int* pos3, int* k_len, cudaStream_t s) {
  gen_rows_kernel<<<nblk((long)B * per_seq), 256, 0, s>>>(len, delta, gen, back, per_seq, B, slot, row0, pages, dest_rows,
                                                          pos3, k_len);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void page_rows(const int* rows, const int* pages, int* out, long n, cudaStream_t s) {
  if (n <= 0) return;
  page_rows_kernel<<<nblk(n), 256, 0, s>>>(rows, pages, out, n);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void kv_append(const bf16* qkv, int ld, int k_off, int v_off, int kvdim, const int* dest_rows, long rows, bf16* cache_k,
               bf16* cache_v, cudaStream_t s) {
  N1_CHECK(kvdim % 8 == 0 && ld % 8 == 0 && k_off % 8 == 0 && v_off % 8 == 0, "kv_append: alignment");
  if (rows <= 0) return;
  kv_append_kernel<<<nblk(rows * (kvdim / 8)), 256, 0, s>>>(qkv, ld, k_off, v_off, kvdim / 8, dest_rows, rows, cache_k,
                                                           cache_v);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void latent_src(const int* cur_tok, int B, int nq, int* kind, int* src, cudaStream_t s) {
  latent_src_kernel<<<nblk((long)B * (nq + 1)), 256, 0, s>>>(cur_tok, B, nq, kind, src);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void argmax_rows(const bf16* logits, long ld, int n, int rows, int* out, cudaStream_t s) {
  argmax_rows_kernel<<<rows, 256, 0, s>>>(logits, ld, n, out);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}
void gen_update(const int* next, int* cur_tok, int* gen, int* finished, int* out_tokens, int max_new, const int* eos,
                int n_eos, int B, int* n_active, cudaStream_t s) {
  N1_CHECK(n_eos >= 0 && n_eos <= 4, "gen_update: at most 4 eos ids");
  int e[4] = {-1, -1, -1, -1};
  for (int i = 0; i < n_eos; ++i) e[i] = eos[i];
  N1_CUDA(cudaMemsetAsync(n_active, 0, sizeof(int), s));
  gen_update_kernel<<<nblk(B), 256, 0, s>>>(next, cur_tok, gen, finished, out_tokens, max_new, e[0], e[1], e[2], e[3], B,
                                            n_active);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

void image_digest(const bf16* pixels, long cols, const int64_t* row_off, int n_img, uint64_t* digest, cudaStream_t s) {
  N1_CHECK(cols % 2 == 0 && n_img >= 0, "image_digest: cols must be even");
  if (n_img == 0) return;
  image_digest_kernel<<<n_img, 256, 0, s>>>(reinterpret_cast<const uint32_t*>(pixels), cols / 2, row_off, digest);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

}  // namespace n1
