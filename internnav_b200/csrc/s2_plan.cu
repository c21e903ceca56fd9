#include "s2_plan.h"

#include <algorithm>
#include <numeric>

#include "n1_ops.h"

namespace n1 {

void vit_index(const int32_t* grid_thw, int n_img, int merge, int win, VitIndex& o) {
  o = VitIndex();
  const int unit = merge * merge;
  std::vector<int> cu_window_raw = {0};
  int window_index_id = 0;
  std::vector<int> pos_src;  // (h, w) per patch in the processor's patch order (merge-block major)
  for (int im = 0; im < n_img; ++im) {
    const int t = grid_thw[im * 3], h = grid_thw[im * 3 + 1], w = grid_thw[im * 3 + 2];
    N1_CHECK(t > 0 && h > 0 && w > 0 && h % merge == 0 && w % merge == 0, "bad image_grid_thw");
    // ---- rot_pos_emb ids: hpos/wpos reshaped (h/m, m, w/m, m) -> permute(0, 2, 1, 3) -> flatten, repeated t times
    for (int rep = 0; rep < t; ++rep)
      for (int bh = 0; bh < h / merge; ++bh)
        for (int bw = 0; bw < w / merge; ++bw)
          for (int ih = 0; ih < merge; ++ih)
            for (int iw = 0; iw < merge; ++iw) {
              pos_src.push_back(bh * merge + ih);
              pos_src.push_back(bw * merge + iw);
            }
    // ---- get_window_index
    const int gh = h / merge, gw = w / merge;
    const int pad_h = win - gh % win, pad_w = win - gw % win;  // NB: a full extra window when already divisible
    const int nwh = (gh + pad_h) / win, nww = (gw + pad_w) / win;
    for (int tt = 0; tt < t; ++tt)
      for (int wh = 0; wh < nwh; ++wh)
        for (int ww = 0; ww < nww; ++ww) {
          int count = 0;
          for (int ih = 0; ih < win; ++ih)
            for (int iw = 0; iw < win; ++iw) {
              const int y = wh * win + ih, x = ww * win + iw;
              if (y < gh && x < gw) {
                o.window_index.push_back(window_index_id + (tt * gh + y) * gw + x);
                ++count;
              }
            }
          cu_window_raw.push_back(cu_window_raw.back() + count * unit);
        }
    window_index_id += t * gh * gw;
    for (int tt = 0; tt < t; ++tt) o.cu_full.push_back(h * w);
    o.n_patches += (long)t * h * w;
  }
  // unique_consecutive
  for (int v : cu_window_raw)
    if (o.cu_window.empty() || o.cu_window.back() != v) o.cu_window.push_back(v);
  // cu_full: cumsum with leading zero
  {
    std::vector<int> c = {0};
    for (int v : o.cu_full) c.push_back(c.back() + v);
    o.cu_full = c;
  }
  for (size_t i = 1; i < o.cu_window.size(); ++i) o.max_window = std::max(o.max_window, o.cu_window[i] - o.cu_window[i - 1]);
  for (size_t i = 1; i < o.cu_full.size(); ++i) o.max_full = std::max(o.max_full, o.cu_full[i] - o.cu_full[i - 1]);
  const int n_merged = (int)o.window_index.size();
  N1_CHECK((long)n_merged * unit == o.n_patches, "window index does not cover all patches");
  o.reverse_index.resize(n_merged);
  for (int i = 0; i < n_merged; ++i) o.reverse_index[o.window_index[i]] = i;  // argsort of a permutation
  // position ids reordered like hidden_states[window_index] on groups of `unit` patches
  o.pos_hw.resize(o.n_patches * 2);
  for (int i = 0; i < n_merged; ++i)
    for (int u = 0; u < unit; ++u) {
      const long dst = (long)i * unit + u, src = (long)o.window_index[i] * unit + u;
      o.pos_hw[dst * 2] = pos_src[src * 2];
      o.pos_hw[dst * 2 + 1] = pos_src[src * 2 + 1];
    }
}

void rope_index_one(const int32_t* ids, int len, const int32_t* grid_thw, int n_img, int merge, int& cursor,
                    std::vector<int>& pos3, int& delta) {
  pos3.assign((size_t)3 * len, 0);
  int image_nums = 0;
  for (int i = 0; i + 1 < len; ++i)
    if (ids[i] == kVisionStartId && ids[i + 1] == kImageTokenId) ++image_nums;
  int st = 0;
  int out = 0;          // number of positions written
  int last_max = -1;    // max of the last appended block
  bool any = false;
  auto put = [&](int a, int b, int c) {
    N1_CHECK(out < len, "rope index overflow (image tokens do not match image_grid_thw)");
    pos3[out] = a, pos3[len + out] = b, pos3[2 * len + out] = c;
    ++out;
  };
  for (int n = 0; n < image_nums; ++n) {
    int ed = -1;
    for (int i = st; i < len; ++i)
      if (ids[i] == kImageTokenId) {
        ed = i;
        break;
      }
    N1_CHECK(ed >= 0, "image token not found");
    N1_CHECK(cursor < n_img, "more image placeholders than rows in image_grid_thw");
    const int t = grid_thw[cursor * 3], h = grid_thw[cursor * 3 + 1] / merge, w = grid_thw[cursor * 3 + 2] / merge;
    ++cursor;
    const int text_len = ed - st;
    const int st_idx = any ? last_max + 1 : 0;
    for (int i = 0; i < text_len; ++i) put(i + st_idx, i + st_idx, i + st_idx);
    // images: second_per_grid_t = 0 -> temporal index 0 for every frame
    for (int tt = 0; tt < t; ++tt)
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) put(0 + text_len + st_idx, y + text_len + st_idx, x + text_len + st_idx);
    last_max = std::max(h, w) - 1 + text_len + st_idx;
    if (text_len > 0 && t * h * w == 0) last_max = text_len - 1 + st_idx;
    any = true;
    st = ed + t * h * w;
  }
  if (st < len) {
    const int st_idx = any ? last_max + 1 : 0;
    const int text_len = len - st;
    for (int i = 0; i < text_len; ++i) put(i + st_idx, i + st_idx, i + st_idx);
    last_max = text_len - 1 + st_idx;
    any = true;
  }
  N1_CHECK(out == len, "rope index: sequence length mismatch");
  int mx = 0;
  for (int v : pos3) mx = std::max(mx, v);
  delta = mx + 1 - len;
}

void plan_rows(const int32_t* ids, const int32_t* lens, int B, const int32_t* grid, int n_img, const PlanArgs& a,
               PlanRows& o) {
  o = PlanRows();
  const bool cont = a.ctx != nullptr, gen = a.max_new > 0;
  N1_CHECK(cont == (a.slots != nullptr), "continuation plan: ctx and slots go together");
  N1_CHECK(!cont || gen, "continuation plan: only generation plans continue a cache");
  const int nq = gen ? 0 : a.n_query, unit = a.merge * a.merge;
  if (cont) {
    std::vector<char> used(a.pool_slots, 0);
    for (int b = 0; b < B; ++b) {
      N1_CHECK(a.slots[b] >= 0 && a.slots[b] < a.pool_slots, "continuation plan: slot " + std::to_string(a.slots[b]) +
                                                                 " out of range [0, " + std::to_string(a.pool_slots) + ")");
      N1_CHECK(!used[a.slots[b]], "continuation plan: slot " + std::to_string(a.slots[b]) + " used twice in one batch");
      used[a.slots[b]] = 1;
      N1_CHECK(a.ctx[b] >= 0 && a.ctx[b] < lens[b], "continuation plan: reused length must be in [0, prompt length)");
      const int limit = a.pool_limit > 0 ? a.pool_limit : a.pool_cap;
      N1_CHECK((long)lens[b] + a.max_new + a.n_query <= limit,
               "continuation plan: prompt + max_new_tokens + n_query exceeds the pool's slot capacity (" +
                   std::to_string(limit) + ")");
      o.ctx.push_back(a.ctx[b]), o.slot_of.push_back(a.slots[b]);
      o.any_ctx |= a.ctx[b] > 0;
    }
  }
  o.cu.push_back(0);
  int cursor = 0;
  long off = 0, expect_cont = 0;
  std::vector<std::vector<int>> pos_seq(B);
  for (int b = 0; b < B; ++b) {
    const int len = lens[b];
    N1_CHECK(len > 0, "empty prompt");
    std::vector<int> seq(ids + off, ids + off + len);
    off += len;
    for (int q = 0; q < nq; ++q) seq.push_back(kTrajTokenId);  // internvla_n1.py L327
    const int L = (int)seq.size();
    const int c = cont ? a.ctx[b] : 0;
    const int first_img = cursor;
    int delta = 0;
    rope_index_one(seq.data(), L, grid, n_img, a.merge, cursor, pos_seq[b], delta);
    o.delta.push_back(delta);
    if (cont) {  // images of this prompt: those wholly before c were prefilled before, none may straddle c
      int im = first_img;
      for (int i = 0; i < L; ++i)
        if (seq[i] == kImageTokenId && (i == 0 || seq[i - 1] != kImageTokenId)) {
          N1_CHECK(im < cursor, "image placeholder without a grid row");
          const int n = grid[im * 3] * grid[im * 3 + 1] * grid[im * 3 + 2] / unit;
          N1_CHECK(!(i < c && c < i + n), "continuation plan: the reused prefix would end inside an image");
          if (i >= c) expect_cont += n;
          ++im;
        }
    }
    for (int i = c; i < L; ++i) {
      if (i >= len) {
        o.kind.push_back(2), o.src.push_back(i - len);  // latent_queries[q]
        o.out_rows.push_back((int)o.kind.size() - 1);
      } else if (seq[i] == kImageTokenId) {
        o.kind.push_back(1), o.src.push_back((int)o.n_image_tokens++);  // image features in order (L332)
      } else {
        N1_CHECK(seq[i] >= 0 && seq[i] < a.vocab, "token id out of vocabulary");
        o.kind.push_back(0), o.src.push_back(seq[i]);
      }
    }
    if (gen) o.out_rows.push_back((int)o.kind.size() - 1);  // logits of the last prompt token start the decode
    o.cu.push_back(o.cu.back() + L - c);
    o.max_len = std::max(o.max_len, L - c);
    if (c > 0) {  // keep the positions of rows [c, L) ([3, L - c])
      std::vector<int> t((size_t)3 * (L - c));
      for (int st = 0; st < 3; ++st)
        std::copy(pos_seq[b].begin() + (size_t)st * L + c, pos_seq[b].begin() + (size_t)(st + 1) * L,
                  t.begin() + (size_t)st * (L - c));
      pos_seq[b].swap(t);
    }
  }
  const long tokens = o.cu.back();
  long expect = 0;
  for (int i = 0; i < cursor; ++i) expect += (long)grid[i * 3] * grid[i * 3 + 1] * grid[i * 3 + 2] / unit;
  if (cont) expect = expect_cont;
  N1_CHECK(expect == o.n_image_tokens, "Image features and image tokens do not match: tokens " +
                                           std::to_string(o.n_image_tokens) + ", features " +
                                           std::to_string(expect));  // same check as internvla_n1.py L135-138
  // [3, tokens] layout over the packed batch
  o.pos3.assign((size_t)3 * tokens, 0);
  for (int b = 0; b < B; ++b) {
    const int L = o.cu[b + 1] - o.cu[b];
    for (int st = 0; st < 3; ++st)
      for (int i = 0; i < L; ++i) o.pos3[(size_t)st * tokens + o.cu[b] + i] = pos_seq[b][(size_t)st * L + i];
  }
  if (gen) {
    o.slot = cont ? a.pool_cap : o.max_len + a.max_new + a.n_query;
    o.dest.resize(tokens), o.len.resize(B);
    for (int b = 0; b < B; ++b) {
      const int n = o.cu[b + 1] - o.cu[b], c = cont ? a.ctx[b] : 0;
      const int r0 = cont ? a.slots[b] * a.pool_cap : b * o.slot;
      o.len[b] = c + n;
      for (int i = 0; i < n; ++i) o.dest[o.cu[b] + i] = r0 + c + i;
      if (cont) o.row0.push_back(r0);
    }
  }
}

void PageAlloc::init(int s, int ps, int n) {
  N1_CHECK(s > 0 && ps > 0 && n > 0 && (long)s * ps < (1L << 31) && (long)n * kPageRows < (1L << 31),
           "kv pages: slots, pages per slot and pages must be positive");
  slots = s, per_slot = ps, pages = n;
  table.assign((size_t)s * ps, -1);
  held.assign(s, 0);
  free.resize(n);
  for (int i = 0; i < n; ++i) free[i] = n - 1 - i;  // page 0 on top
}

std::pair<int, int> PageAlloc::prepare(int B, const int32_t* slot, const int32_t* keep_rows, const int32_t* need_rows) {
  auto pages_of = [](long rows) { return (int)((rows + kPageRows - 1) / kPageRows); };
  long give = 0, take = 0;
  std::vector<char> seen(slots, 0);
  for (int b = 0; b < B; ++b) {
    const int s = slot[b];
    N1_CHECK(s >= 0 && s < slots && !seen[s], "kv pages: slot " + std::to_string(s) + " out of range or used twice");
    seen[s] = 1;
    const int keep = pages_of(keep_rows[b]), need = pages_of(need_rows[b]);
    N1_CHECK(keep_rows[b] >= 0 && keep <= held[s] && keep_rows[b] <= need_rows[b] && need <= per_slot,
             "kv pages: sequence " + std::to_string(b) + " keeps " + std::to_string(keep_rows[b]) + " of the " +
                 std::to_string(held[s] * kPageRows) + " rows its slot holds and needs " + std::to_string(need_rows[b]) +
                 " (at most " + std::to_string(per_slot * kPageRows) + ")");
    give += held[s] - keep, take += need - keep;
  }
  if (take > (long)free.size() + give)
    throw Error(kErrKvPages, "kv pages: the call needs " + std::to_string(take) + " pages, " +
                                 std::to_string(free.size() + give) + " are free (" + std::to_string(free.size()) +
                                 " in the pool, " + std::to_string(give) + " returned by the call's own slots)");
  for (int b = 0; b < B; ++b) trim(slot[b], keep_rows[b]);
  int lo = slots, hi = 0;
  for (int b = 0; b < B; ++b) {
    const int s = slot[b], need = pages_of(need_rows[b]);
    if (held[s] >= need) continue;
    for (int* t = &table[(size_t)s * per_slot]; held[s] < need; ++held[s]) {
      t[held[s]] = free.back();
      free.pop_back();
    }
    lo = std::min(lo, s), hi = std::max(hi, s + 1);
  }
  return lo < hi ? std::make_pair(lo, hi) : std::make_pair(0, 0);
}

void PageAlloc::trim(int s, int rows) {
  N1_CHECK(s >= 0 && s < slots && rows >= 0, "kv pages: slot out of range");
  const int keep = (int)(((long)rows + kPageRows - 1) / kPageRows);
  int* t = &table[(size_t)s * per_slot];
  for (; held[s] > keep; --held[s]) {  // last page first, so the slot's first page ends on top of the free list
    free.push_back(t[held[s] - 1]);
    t[held[s] - 1] = -1;
  }
}

}  // namespace n1
