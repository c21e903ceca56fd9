// System-2 executor: Qwen2.5-VL vision transformer and decoder prefill, sequenced from host C++ over the kernels in
// this directory.  Replaces `self.visual(pixel_values, grid_thw)` and `self.model(inputs_embeds, position_ids)` as
// called by InternVLAN1ForCausalLM.generate_latents (internvla_n1.py L320-347); the arithmetic itself lives in the
// un-vendored pin transformers==4.51.0 (modeling_qwen2_5_vl.py) and is restated in oracle/qwen_oracle.py.
#pragma once
#include <vector>

#include "s1_model.h"
#include "s2_plan.h"

namespace n1 {

struct S2Dims {
  // vision tower
  int v_depth = 32, v_hidden = 1280, v_heads = 16, v_inter = 3420, v_patch = 14, v_tpatch = 2, v_merge = 2;
  int v_window = 112, v_out = 3584;
  int n_fullatt = 4, fullatt[16] = {7, 15, 23, 31};
  // language model
  int layers = 28, hidden = 3584, heads = 28, kv_heads = 4, head_dim = 128, inter = 18944, vocab = 152064;
  float rms_eps = 1e-6f, rope_theta = 1000000.0f;
  int mrope[3] = {16, 24, 24};
  int n_query = 4;
};

// Device-resident index arrays for one batch of images (immutable; reusable across calls with the same grids).
struct VitPlan {
  VitIndex host;
  int *window_index = nullptr, *reverse_index = nullptr, *cu_window = nullptr, *cu_full = nullptr;
  float2* rope = nullptr;  // [n_patches, head_dim / 2] (cos, sin), window order
  int n_window = 0, n_full = 0;
  ~VitPlan();
};

// Caller-owned K/V cache pool: `slots` conversations of up to `cap` rows each, per decoder layer.  Sized once
// (n1_kv_pool_create) and never reallocated by a hot call.  valid[s] = rows of slot s whose K/V a pass actually wrote
// for the conversation's tokens (prompt + generated; never the TRAJ rows of the latent pass).
// A paged pool (n1_kv_pool_create_paged) holds `pages` pages of 64 rows instead, any of which serves any slot: plans
// still address slot s at rows s * cap + i (cap = max_pages * 64), and `table` maps such a row to pool row
// table[row / 64] * 64 + row % 64.  The host PageAlloc is authoritative; llm_generate uploads the rows it changes.
struct KvPool {
  bf16 *k = nullptr, *v = nullptr;  // [layers][rows()][width]
  int slots = 0, cap = 0;
  long layer_stride = 0;
  std::vector<int> valid;
  size_t bytes() const { return 2 * (size_t)layer_stride * layers * sizeof(bf16); }
  int layers = 0, width = 0;  // width = kv_heads * head_dim
  // paged pools only
  int max_tokens = 0;       // rows one conversation may hold (the plan bound)
  int* table = nullptr;     // device [slots][cap / 64]
  PageAlloc pages;
  bool paged() const { return table != nullptr; }
  long rows() const { return layer_stride / width; }
  ~KvPool();
};

// Device-resident token bookkeeping for one batch of prompts (generate_latents appends n_query TRAJ tokens each).
struct LlmPlan {
  int B = 0, max_len = 0, n_query = 0;
  int n_out = 0;  // rows read after the last layer: B * n_query TRAJ rows (latent plan) or the B last prompt rows
  long tokens = 0, n_image_tokens = 0;
  std::vector<int> h_cu, h_pos3, h_delta;
  int *cu = nullptr, *kind = nullptr, *src = nullptr, *out_rows = nullptr;
  float2* rope = nullptr;  // [tokens, head_dim / 2]
  // generation plans only (max_new > 0): every sequence owns `slot` rows of the per-layer K/V cache
  int max_new = 0, slot = 0;
  int *dest_rows = nullptr, *d_len = nullptr, *d_delta = nullptr;  // [tokens], [B], [B]
  // continuation plans only (pool != nullptr): sequence b reuses the first ctx[b] rows of pool slot h_slot[b]; the plan's
  // rows are the suffix [ctx[b], len[b]) of each prompt, and its K/V live in the pool (first row row0[b])
  KvPool* pool = nullptr;
  std::vector<int> h_ctx, h_slot, h_len;
  int *ctx = nullptr, *row0 = nullptr;
  bool any_ctx = false;  // some sequence reuses rows: the prefill attends through the pool (attention_cache)
  // All device arrays above are carved from ONE pooled block (plan_pool in s2_model.cu): a plan is created every policy
  // step (prompts change), so creation must not cudaMalloc / cudaFree / synchronise once the pool is warm.  `ready` is
  // recorded after the upload + RoPE-table kernel on the creating stream; `last_use` after every hot call, so a recycled
  // block is never overwritten while a consumer on another stream may still read it.
  void* block = nullptr;
  size_t block_bytes = 0;
  cudaEvent_t ready = nullptr;
  mutable cudaEvent_t last_use = nullptr;
  void wait_ready(cudaStream_t s) const;  // first statement of every hot call
  void mark_used(cudaStream_t s) const;   // last statement of every hot call
  ~LlmPlan();
};

// Result of one greedy generation (host side of n1_llm_generate).
struct GenResult {
  int32_t* tokens = nullptr;  // host [B, max_new], unfilled entries = pad
  int32_t* lens = nullptr;    // host [B]
  int steps = 0;              // decode passes executed after the prefill
};

class S2Model {
 public:
  S2Dims dims;
  void load(const WeightSource& ws, const S2Dims& d, cudaStream_t s);
  bool loaded() const { return loaded_; }

  VitPlan* make_vit_plan(const int32_t* grid_thw_host, int n_img, cudaStream_t s) const;
  // ids: packed prompt token ids (host), lens[B].
  // max_new_tokens 0: latent plan (generate_latents; TRAJ tokens are appended per sequence by the planner).  >= 1:
  // generation plan (no TRAJ tokens; KV-cache slots sized for the prompt + max_new_tokens + n_query rows).
  // ctx_host / slot_host / pool (all or none; generation plans only): a continuation plan over the FULL prompts and all
  // their image grids (mRoPE positions come from the whole prompt) that embeds and prefills rows [ctx[b], len[b]) only;
  // image features are expected for the images whose tokens lie in those rows, and no image may straddle ctx[b].
  LlmPlan* make_llm_plan(const int32_t* ids_host, const int32_t* lens_host, int B, const int32_t* grid_thw_host,
                         int n_img, cudaStream_t s, int max_new_tokens, const int32_t* ctx_host, const int32_t* slot_host,
                         KvPool* pool) const;
  KvPool* make_pool(int slots, int cap) const;
  KvPool* make_paged_pool(int slots, int pages, int max_tokens_per_slot) const;

  size_t ws_vit(const VitPlan& p) const;
  // pixels bf16 [n_patches, 3 * tpatch * patch^2] -> out bf16 [n_patches / merge^2, v_out] (original token order).
  // dst_rows_host (host, n_patches / merge^2 entries, checked by the caller): merged row r goes to out[dst_rows_host[r]].
  void vit_forward(const VitPlan& p, void* ws, size_t ws_bytes, const bf16* pixels, bf16* out, cudaStream_t s,
                   const int32_t* dst_rows_host) const;
  size_t ws_llm(const LlmPlan& p) const;
  // image_feats bf16 [n_image_tokens, hidden] -> out bf16 [B, n_query, hidden] (final-norm states of the TRAJ rows)
  void llm_prefill(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* image_feats, bf16* out,
                   cudaStream_t s) const;
  // Greedy decode (model.generate(do_sample=False), internvla_n1_policy.py L169-176) on a generation plan: prefill with
  // K/V kept per layer, then one token per pass until every sequence emitted an eos id or max_new tokens.  When
  // `latents` is non-null the cache is reused for generate_latents(output_ids, ...) (internvla_n1.py L320-347): one more
  // pass over [last token, TRAJ x n_query] per sequence -> latents bf16 [B, n_query, hidden].  Synchronises `s`.
  // image_rows_host (host, n_image_tokens entries, checked by the caller): image token i reads image_feats row
  // image_rows_host[i] instead of row i (image_feats is then a feature pool).
  // On a continuation plan K/V are read from and written to the plan's pool, and pool->valid is updated.
  size_t ws_generate(const LlmPlan& p) const;
  void llm_generate(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* image_feats, const int32_t* eos, int n_eos,
                    int32_t pad, GenResult& out, bf16* latents, cudaStream_t s, const int32_t* image_rows_host) const;
  bool has_lm_head() const { return lm_head_.w != nullptr; }
  // optional ("model.latent_queries"); every call that embeds TRAJ rows needs it and refuses to run without it
  bool has_latent_queries() const { return latentq_ != nullptr; }

  // ---- training branch, System-2 half (s2_train.cu)
  // The decoder is frozen and causal: the TRAJ rows are a chunk appended to the prompt's K/V cache (exactly the latent
  // pass of llm_generate), and d loss / d latent_queries needs the backward of those n_query rows per sample only
  // (oracle/qwen_backward.py).  Both calls take a GENERATION plan over the prompts (without TRAJ tokens) and the SAME
  // workspace: the forward leaves the cache and the per-layer TRAJ-row tensors there for the backward.
  // overwrite the library's copy of `latent_queries` (bf16 [n_query, hidden], device) after an optimizer step
  void set_latent_queries(const bf16* src, cudaStream_t s);
  // Refuses a continuation plan (one created over a K/V pool: its rows live in the pool, not in the workspace's cache).
  // train_forward and train_backward size their workspace here before they launch anything, so they refuse it too.
  size_t ws_train(const LlmPlan& p) const;
  // -> states bf16 [B, n_query, hidden] = hidden_states[b, t_s_pos[b] : t_s_pos[b] + n_query] (internvla_n1.py L231-235)
  void train_forward(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* image_feats, bf16* states, cudaStream_t s);
  // grad_states bf16 [B, n_query, hidden] -> grad_latent fp32 [n_query, hidden] (summed over the batch)
  void train_backward(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* grad_states, float* grad_latent,
                      cudaStream_t s);

 private:
  struct KvCache {
    bf16 *k = nullptr, *v = nullptr;  // [layers][B * slot][kv_heads * head_dim]
    long layer_stride = 0;
  };
  // decode-state buffers of gen_impl; the training forward carves the chunk's share of them (s2_train.cu)
  struct GenBufs {
    int *cur_tok = nullptr, *gen = nullptr, *finished = nullptr, *next = nullptr, *k_len = nullptr, *n_active = nullptr;
    int *out_tokens = nullptr, *dest = nullptr, *pos3 = nullptr, *kind = nullptr, *src = nullptr;
    float2* rope = nullptr;
    bf16 *x = nullptr, *ln = nullptr, *qkv = nullptr, *att = nullptr, *hid = nullptr, *normed = nullptr, *logits = nullptr;
  };
  // per-layer tensors of a chunk pass that the training backward reads: layer l's R rows start at row l * R
  struct ChunkSaves {
    bf16 *x_in = nullptr, *qkv = nullptr, *att = nullptr, *x_mid = nullptr;  // layer input, q|k|v, attention, post-attention
  };
  // weights of one pre-norm block, vision tower and decoder alike
  struct Block {
    float *n1 = nullptr, *n2 = nullptr;
    Lin qkv, o, gateup, down;
  };
  // One pre-norm block, split around the step that differs per pass (K/V append and attention); x [rows, H] is the
  // residual stream.  block_in: ln = RMSNorm(x); qkv = linear(ln); RoPE on its first rot_heads heads (q and k).
  static void block_in(const Block& b, const bf16* x, bf16* ln, bf16* qkv, const float2* rope, int rows, int H,
                       int rot_heads, int hd, float eps, cudaStream_t s);
  // block_out: x += linear(att); save_mid (if set) = x; x += down(SwiGLU(gateup(RMSNorm(x)))), hid [rows, inter_pad]
  static void block_out(const Block& b, const bf16* att, bf16* x, bf16* ln, bf16* hid, int rows, int H, int inter_pad,
                        float eps, cudaStream_t s, bf16* save_mid = nullptr);
  // causal attention of per_seq new rows per sequence (packed q|k|v rows) on one layer's slotted K/V cache
  AttnParams cache_attn(const LlmPlan& p, int per_seq, const int* k_len, const bf16* qkv, const bf16* k, const bf16* v,
                        bf16* o) const;
  size_t vit_impl(Carver c, const VitPlan& p, const bf16* pixels, bf16* out, cudaStream_t s,
                  const int32_t* dst_rows_host = nullptr) const;
  size_t llm_impl(Carver c, const LlmPlan& p, const bf16* image_feats, bf16* out, cudaStream_t s,
                  const KvCache* kv = nullptr, const int32_t* image_rows_host = nullptr) const;
  size_t gen_impl(Carver c, const LlmPlan& p, const bf16* image_feats, const int32_t* eos, int n_eos, int32_t pad,
                  GenResult* out, bf16* latents, cudaStream_t s, const int32_t* image_rows_host = nullptr) const;
  void chunk_pass(const GenBufs& g, const LlmPlan& p, const KvCache& kv, int per_seq, cudaStream_t s,
                  const ChunkSaves* save = nullptr) const;

  Arena arena_;
  bool loaded_ = false;
  int v_inter_pad_ = 0, inter_pad_ = 0, patch_k_ = 0;
  Lin v_patch_;
  std::vector<Block> vblk_;
  float* merger_ln_ = nullptr;
  Lin merger0_, merger2_;
  bf16* embed_ = nullptr;    // [vocab, hidden]
  bf16* latentq_ = nullptr;  // [n_query, hidden]; null for a System-2-only checkpoint
  std::vector<Block> lblk_;
  float* final_norm_ = nullptr;
  Lin lm_head_;  // optional ("lm_head.weight"); only generate() needs it
  // transposed copies of the frozen decoder weights for the dgrad GEMMs of train_backward (built on first use; no norms)
  std::vector<Block> lblk_t_;
  struct TrainBufs;
  size_t train_carve(Carver& c, const LlmPlan& p, TrainBufs& t) const;
  void ensure_transposed(cudaStream_t s);
};

}  // namespace n1
