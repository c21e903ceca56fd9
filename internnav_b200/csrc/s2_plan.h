// Host-side integer planning for the System-2 path: everything the reference derives from `input_ids` and
// `image_grid_thw` with Python loops, restated in C++ (bit-exact integer work, SURVEY.md §8 row a4):
//   * get_rope_index  (images only)     -- internnav/dataset/rope2d.py L6-181 == HF Qwen2_5_VLModel.get_rope_index
//   * rot_pos_emb position ids, get_window_index, cu_seqlens -- transformers modeling_qwen2_5_vl.py
//     (Qwen2_5_VisionTransformerPretrainedModel.rot_pos_emb / get_window_index / forward)
#pragma once
#include <stdint.h>

#include <utility>
#include <vector>

namespace n1 {

constexpr int kImageTokenId = 151655;   // IMAGE_TOKEN_INDEX, internvla_n1.py L19
constexpr int kVideoTokenId = 151656;
constexpr int kVisionStartId = 151652;
constexpr int kTrajTokenId = 151667;    // TRAJ_TOKEN_INDEX, internvla_n1.py L18

struct VitIndex {
  long n_patches = 0;                 // sum t*h*w
  std::vector<int> window_index;      // [n_patches / merge^2] merged-token order -> source merged token
  std::vector<int> reverse_index;     // argsort(window_index)
  std::vector<int> cu_window;         // unique_consecutive(cu_window_seqlens), in patches
  std::vector<int> cu_full;           // per (image, frame) sequence boundaries, in patches
  std::vector<int> pos_hw;            // [n_patches, 2] (h, w) ids in WINDOW order
  int max_window = 0, max_full = 0;
};
// grid_thw: [n_img, 3] (t, h, w) in patches.  merge = spatial_merge_size, window = window_size / merge / patch_size.
void vit_index(const int32_t* grid_thw, int n_img, int merge, int vit_merger_window, VitIndex& out);

// One sequence: position ids [3, len] and the mrope delta.  `cursor` = index of the next unused image in grid_thw
// (advanced), matching the reference's running image_index across the batch.
void rope_index_one(const int32_t* ids, int len, const int32_t* grid_thw, int n_img, int merge, int& cursor,
                    std::vector<int>& pos3, int& delta);

// Token bookkeeping of one decoder plan over B packed prompts (all host integer work of S2Model::make_llm_plan).
//   max_new 0: latent plan (n_query TRAJ tokens appended per prompt); >= 1: generation plan, K/V rows of sequence b at
//   b * slot + i with slot = max_len + max_new + n_query.
//   ctx / slots (continuation plan, generation only): sequence b reuses the first ctx[b] rows of pool slot slots[b]
//   (pool_slots x pool_cap rows); its rows are [ctx[b], len[b]) only, their K/V rows slots[b] * pool_cap + i, and image
//   features are expected for the images after ctx[b] alone.
struct PlanArgs {
  int merge = 2, vocab = 0, n_query = 0, max_new = 0;
  const int32_t* ctx = nullptr;
  const int32_t* slots = nullptr;
  int pool_slots = 0, pool_cap = 0;
  int pool_limit = 0;  // rows one conversation may hold (prompt + max_new + n_query); 0: pool_cap
};
struct PlanRows {
  std::vector<int> cu;                  // [B + 1] planned rows per sequence, packed
  std::vector<int> kind, src;           // [rows] 0 text (src = token id), 1 image (src = feature row), 2 latent query
  std::vector<int> out_rows;            // rows read after the last layer
  std::vector<int> pos3;                // [3, rows] mRoPE positions
  std::vector<int> delta;               // [B] mRoPE delta
  std::vector<int> dest, len;           // generation plans: [rows] K/V cache row, [B] keys after the prefill (= prompt length)
  std::vector<int> ctx, slot_of, row0;  // continuation plans: [B] reused rows, pool slot, first K/V row of the slot
  long n_image_tokens = 0;
  int max_len = 0, slot = 0;
  bool any_ctx = false;
};
void plan_rows(const int32_t* ids, const int32_t* lens, int B, const int32_t* grid, int n_img, const PlanArgs& a,
               PlanRows& o);

// Page accounting of a paged K/V pool: `pages` pages of kPageRows rows shared by `slots` conversations of at most
// per_slot pages each.  table[s * per_slot + i] is the pool page that holds rows [i * 64, i * 64 + 64) of slot s (-1: none);
// a slot always holds pages 0 .. held[s] - 1 of its table row, so a plan's rows (slot s at s * per_slot * 64 + position)
// map to pool rows through the table alone.  Freed pages go on top of the free list and are taken from there first.
constexpr int kPageRows = 64;  // = the key block of attn_kernel and attn_cache_kernel: one block is one page
constexpr int kErrKvPages = -8;  // N1_ERR_KV_PAGES
struct PageAlloc {
  int slots = 0, per_slot = 0, pages = 0;
  std::vector<int> table, held, free;
  void init(int slots, int per_slot, int pages);
  // Sequence b (slot slot[b], slots distinct) keeps the pages covering its first keep_rows[b] rows, returns its other
  // pages and takes pages up to need_rows[b] rows.  Throws Error(kErrKvPages) with the pages needed and free, leaving
  // every table unchanged, if they do not fit.  -> [lo, hi): the slots whose table rows changed (lo == hi: none).
  std::pair<int, int> prepare(int B, const int32_t* slot, const int32_t* keep_rows, const int32_t* need_rows);
  void trim(int slot, int rows);  // return the pages past ceil(rows / 64)
  int free_pages() const { return (int)free.size(); }
};

}  // namespace n1
