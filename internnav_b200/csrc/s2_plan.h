// Host-side integer planning for the System-2 path: everything the reference derives from `input_ids` and
// `image_grid_thw` with Python loops, restated in C++ (bit-exact integer work, SURVEY.md §8 row a4):
//   * get_rope_index  (images only)     -- internnav/dataset/rope2d.py L6-181 == HF Qwen2_5_VLModel.get_rope_index
//   * rot_pos_emb position ids, get_window_index, cu_seqlens -- transformers modeling_qwen2_5_vl.py
//     (Qwen2_5_VisionTransformerPretrainedModel.rot_pos_emb / get_window_index / forward)
#pragma once
#include <stdint.h>

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

}  // namespace n1
