// Launchers for the System-2 (Qwen2.5-VL) glue kernels (s2_kernels.cu).
#pragma once
#include "n1_ops.h"

namespace n1 {

// dst[r, :] = src[idx[r / group] * group + r % group, :]   (rows of `cols` bf16; cols % 8 == 0).  With dst_idx the
// destination row is dst_idx[r / group] * group + r % group instead (rows of a caller's feature pool).
void gather_rows(const bf16* src, const int* idx, bf16* dst, long rows, int group, int cols, cudaStream_t s,
                 const int* dst_idx = nullptr);
// ViT 2-D rotary tables: cs[tok, j] = (cos, sin)(pos[tok, j < half/2 ? 0 : 1] * theta^(-2 (j % (half/2)) / half)),
// j in [0, half), half = head_dim / 2.
void vit_rope_table(const int* pos_hw, float2* cs, long tokens, int half, float theta, cudaStream_t s);
// LLM multimodal rotary tables: cs[tok, j] = (cos, sin)(pos[stream(j)][tok] * theta^(-2 j / hd)), j in [0, hd/2);
// stream(j) from mrope_section (t, h, w widths summing to hd/2); pos is [3, tokens] int32.
void mrope_table(const int* pos3, float2* cs, long tokens, int half, int sec_t, int sec_h, float theta, cudaStream_t s);
// In-place rotate-half rotary on the first `heads` heads (each `hd` wide) of every row of x (row stride ld):
// out[j] = x[j] c_j - x[j + hd/2] s_j ; out[j + hd/2] = x[j + hd/2] c_j + x[j] s_j, tables shared by all heads.
void apply_rope(bf16* x, int ld, const float2* cs, long tokens, int heads, int hd, cudaStream_t s);
// LLM input embeddings: kind[tok] 0 -> embed_tokens[src[tok]], 1 -> image_feats[src[tok]], 2 -> latent_queries[src[tok]]
// With image_rows, image tokens read image_feats[image_rows[src[tok]]] (rows of a caller's feature pool).
void build_embeds(const int* kind, const int* src, const bf16* embed_tokens, const bf16* image_feats,
                  const bf16* latent_queries, bf16* out, long tokens, int H, cudaStream_t s,
                  const int* image_rows = nullptr);

// ---- greedy decode with a KV cache (model.generate of internvla_n1_policy.py L169-176, then generate_latents reusing it)
// Chunk bookkeeping: per sequence the tokens idx = len + gen - back + j (j < per_seq) -> cache rows b * slot + idx
// (row0[b] + idx when row0 is given: a slot of a K/V pool; a row r of that is pool row pages[r / 64] * 64 + r % 64 when
// the pool is paged), mrope positions idx + delta on all three axes ([3, B * per_seq]), k_len[b] = last idx + 1.
void gen_rows(const int* len, const int* delta, const int* gen, int back, int per_seq, int B, int slot, const int* row0,
              const int* pages, int* dest_rows, int* pos3, int* k_len, cudaStream_t s);
// out[i] = pages[rows[i] / 64] * 64 + rows[i] % 64: a plan's K/V rows (slot s at s * cap + position) -> paged pool rows
void page_rows(const int* rows, const int* pages, int* out, long n, cudaStream_t s);
// cache_k/v[dest_rows[r], :] = qkv[r, k_off / v_off : + kvdim]
void kv_append(const bf16* qkv, int ld, int k_off, int v_off, int kvdim, const int* dest_rows, long rows, bf16* cache_k,
               bf16* cache_v, cudaStream_t s);
// build_embeds sources of the latent pass: per sequence [embed_tokens[cur_tok], latent_queries[0..nq)]
void latent_src(const int* cur_tok, int B, int nq, int* kind, int* src, cudaStream_t s);
// out[r] = first index of the maximum of logits[r, 0:n]  (torch.argmax tie rule)
void argmax_rows(const bf16* logits, long ld, int n, int rows, int* out, cudaStream_t s);
// Append next[b] to every unfinished sequence; eos (host array, <= 4 ids) or gen == max_new finishes it.
void gen_update(const int* next, int* cur_tok, int* gen, int* finished, int* out_tokens, int max_new, const int* eos_host,
                int n_eos, int B, int* n_active, cudaStream_t s);

// Content digest of n_img images: image i is rows [row_off[i], row_off[i + 1]) of a bf16 [*, cols] matrix (device
// pointers; cols even).  digest[i] = sum over its 32-bit words w at index j of splitmix64(j << 32 | w), plus the word
// count: equal rows give equal digests, and any change of a value or of the row count changes it but with ~2^-64 odds.
void image_digest(const bf16* pixels, long cols, const int64_t* row_off, int n_img, uint64_t* digest, cudaStream_t s);

}  // namespace n1
