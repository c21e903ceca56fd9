// System-2 executor (Qwen2.5-VL ViT + decoder prefill).  See s2_model.h.
#include "s2_model.h"

#include <math.h>
#include <stdlib.h>

#include <string.h>

#include <algorithm>
#include <memory>
#include <mutex>
#include <vector>

#include "s2_kernels.h"

namespace n1 {

namespace {

template <typename T>
T* upload(const std::vector<T>& v, cudaStream_t s) {
  T* d = nullptr;
  N1_CUDA(cudaMalloc(&d, std::max<size_t>(v.size(), 1) * sizeof(T)));
  if (!v.empty()) N1_CUDA(cudaMemcpyAsync(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s));
  return d;
}

// [rows_a; rows_b; ...] stacked into one K-major bf16 matrix (+ optional stacked fp32 bias)
Lin stack_lin(Arena& a, const WeightSource& ws, const std::vector<std::string>& names, bool bias, long cols,
              cudaStream_t s) {
  Lin L;
  long rows = 0;
  for (const std::string& n : names) rows += ws.get(n + ".weight").numel() / cols;
  L.N = (int)rows, L.K = (int)((cols + 7) & ~7L), L.ldw = L.K;
  N1_CHECK(L.N % 8 == 0, "stacked linear: N % 8");
  L.w = a.alloc_n<bf16>((size_t)rows * L.ldw);
  if (bias) L.b = a.alloc_n<float>(rows);
  long r0 = 0;
  for (const std::string& n : names) {
    const SrcTensor& w = ws.get(n + ".weight");
    const long r = w.numel() / cols;
    pack2d(w.data, w.dtype, cols, 0, r, cols, L.w + (size_t)r0 * L.ldw, 1, L.ldw, s);
    if (bias) {
      const SrcTensor& b = ws.get(n + ".bias");
      pack2d(b.data, b.dtype, 1, 0, r, 1, L.b + r0, 0, 1, s);
    }
    r0 += r;
  }
  return L;
}

// SwiGLU pair: rows interleaved (gate_j, up_j), padded to inter_pad zero rows so the GEMM N is a multiple of 16
Lin gateup_lin(Arena& a, const WeightSource& ws, const std::string& p, bool bias, long inter, long inter_pad, long cols,
               cudaStream_t s) {
  Lin L;
  L.N = (int)(2 * inter_pad), L.K = (int)((cols + 7) & ~7L), L.ldw = L.K;
  L.w = a.alloc_n<bf16>((size_t)L.N * L.ldw);
  N1_CUDA(cudaMemsetAsync(L.w, 0, (size_t)L.N * L.ldw * sizeof(bf16), s));
  const SrcTensor& g = ws.get(p + "gate_proj.weight");
  const SrcTensor& u = ws.get(p + "up_proj.weight");
  N1_CHECK(g.numel() == inter * cols && u.numel() == inter * cols, p + "gate/up shape mismatch");
  N1_CHECK(g.dtype == u.dtype, p + "gate/up dtype mismatch");
  interleave_rows(g.data, u.data, g.dtype, inter, cols, L.w, 1, L.ldw, s);
  if (bias) {
    L.b = a.alloc_n<float>(L.N);
    N1_CUDA(cudaMemsetAsync(L.b, 0, L.N * sizeof(float), s));
    const SrcTensor& gb = ws.get(p + "gate_proj.bias");
    const SrcTensor& ub = ws.get(p + "up_proj.bias");
    interleave_rows(gb.data, ub.data, gb.dtype, inter, 1, L.b, 0, 1, s);
  }
  return L;
}

Lin plain_lin(Arena& a, const WeightSource& ws, const std::string& name, bool bias, long rows, long cols,
              cudaStream_t s) {
  Lin L;
  L.N = (int)rows, L.K = (int)((cols + 7) & ~7L);
  L.w = ws.mat(a, name + ".weight", 0, rows, cols, &L.ldw, s);
  if (bias) L.b = ws.f32(a, name + ".bias", s);
  N1_CHECK(L.N % 8 == 0, name + ": N % 8");
  return L;
}

}  // namespace

VitPlan::~VitPlan() {
  cudaFree(window_index), cudaFree(reverse_index), cudaFree(cu_window), cudaFree(cu_full), cudaFree(rope);
}
// ---- pooled plan storage: device blocks (and their pinned staging twins) are recycled across plans
namespace {
struct PlanBlock {
  void* dev = nullptr;
  void* host = nullptr;  // pinned staging of the integer arrays
  size_t bytes = 0;
  cudaEvent_t last_use = nullptr;  // recorded by the previous owner's consumers
};
std::mutex g_pool_mu;
std::vector<PlanBlock> g_pool;

PlanBlock pool_take(size_t bytes) {
  {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    for (size_t i = 0; i < g_pool.size(); ++i)
      if (g_pool[i].bytes >= bytes) {
        PlanBlock b = g_pool[i];
        g_pool.erase(g_pool.begin() + i);
        return b;
      }
  }
  PlanBlock b;
  b.bytes = (bytes + (1 << 20) - 1) & ~size_t((1 << 20) - 1);  // 1 MiB granularity: similar prompts share a size class
  N1_CUDA(cudaMalloc(&b.dev, b.bytes));
  N1_CUDA(cudaMallocHost(&b.host, b.bytes));
  N1_CUDA(cudaEventCreateWithFlags(&b.last_use, cudaEventDisableTiming));
  return b;
}
void pool_give(const PlanBlock& b) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (g_pool.size() < 128) {
    g_pool.push_back(b);
    return;
  }
  cudaFree(b.dev), cudaFreeHost(b.host), cudaEventDestroy(b.last_use);
}
struct PlanHostTwin {  // keeps the pinned twin reachable from the plan without widening the public struct
  std::mutex mu;
  std::vector<std::pair<const void*, void*>> map;
} g_twin;
}  // namespace

void LlmPlan::wait_ready(cudaStream_t s) const {
  if (ready) N1_CUDA(cudaStreamWaitEvent(s, ready, 0));
}
void LlmPlan::mark_used(cudaStream_t s) const {
  if (last_use) N1_CUDA(cudaEventRecord(last_use, s));
}
LlmPlan::~LlmPlan() {
  if (ready) cudaEventDestroy(ready);
  if (block) {
    PlanBlock b;
    b.dev = block, b.bytes = block_bytes, b.last_use = last_use;
    {
      std::lock_guard<std::mutex> lk(g_twin.mu);
      for (size_t i = 0; i < g_twin.map.size(); ++i)
        if (g_twin.map[i].first == block) {
          b.host = g_twin.map[i].second;
          g_twin.map.erase(g_twin.map.begin() + i);
          break;
        }
    }
    pool_give(b);
  }
}

// ------------------------------------------------------------------------------------------------ load
void S2Model::load(const WeightSource& ws, const S2Dims& d, cudaStream_t s) {
  dims = d;
  N1_CHECK(d.v_hidden % d.v_heads == 0 && d.v_hidden / d.v_heads == 80, "vision head_dim must be 80");
  N1_CHECK(d.head_dim == 128 && d.hidden == d.heads * d.head_dim, "decoder head_dim must be 128, hidden = heads * 128");
  N1_CHECK(d.heads % d.kv_heads == 0, "heads % kv_heads");
  N1_CHECK(d.mrope[0] + d.mrope[1] + d.mrope[2] == d.head_dim / 2, "mrope_section must sum to head_dim / 2");
  N1_CHECK(d.v_hidden % 8 == 0 && d.hidden % 8 == 0 && d.v_out == d.hidden, "hidden sizes");
  const WeightSource v = ws.sub("visual.");
  const int Hv = d.v_hidden;
  patch_k_ = 3 * d.v_tpatch * d.v_patch * d.v_patch;
  v_patch_ = plain_lin(arena_, v, "patch_embed.proj", false, Hv, patch_k_, s);
  v_inter_pad_ = (d.v_inter + 7) & ~7;
  vblk_.resize(d.v_depth);
  for (int i = 0; i < d.v_depth; ++i) {
    const std::string p = "blocks." + std::to_string(i) + ".";
    Block& b = vblk_[i];
    b.n1 = v.f32(arena_, p + "norm1.weight", s);
    b.n2 = v.f32(arena_, p + "norm2.weight", s);
    b.qkv = plain_lin(arena_, v, p + "attn.qkv", true, 3 * Hv, Hv, s);
    b.o = plain_lin(arena_, v, p + "attn.proj", true, Hv, Hv, s);
    b.gateup = gateup_lin(arena_, v, p + "mlp.", true, d.v_inter, v_inter_pad_, Hv, s);
    b.down = plain_lin(arena_, v, p + "mlp.down_proj", true, Hv, d.v_inter, s);
    N1_CHECK(b.down.K == v_inter_pad_, "vision down_proj K padding");
  }
  merger_ln_ = v.f32(arena_, "merger.ln_q.weight", s);
  const int unit = d.v_merge * d.v_merge;
  merger0_ = plain_lin(arena_, v, "merger.mlp.0", true, Hv * unit, Hv * unit, s);
  merger2_ = plain_lin(arena_, v, "merger.mlp.2", true, d.v_out, Hv * unit, s);

  const WeightSource m = ws.sub("model.");
  const int H = d.hidden;
  {
    int ld;
    embed_ = m.mat(arena_, "embed_tokens.weight", 0, d.vocab, H, &ld, s);
    // a System-2-only checkpoint (no System 1 in its config) has no latent queries; generate() does not need them
    latentq_ = m.has("latent_queries") ? m.mat(arena_, "latent_queries", 0, d.n_query, H, &ld, s) : nullptr;
  }
  inter_pad_ = (d.inter + 7) & ~7;
  lblk_.resize(d.layers);
  for (int i = 0; i < d.layers; ++i) {
    const std::string p = "layers." + std::to_string(i) + ".";
    Block& b = lblk_[i];
    b.n1 = m.f32(arena_, p + "input_layernorm.weight", s);
    b.n2 = m.f32(arena_, p + "post_attention_layernorm.weight", s);
    b.qkv = stack_lin(arena_, m, {p + "self_attn.q_proj", p + "self_attn.k_proj", p + "self_attn.v_proj"}, true, H, s);
    N1_CHECK(b.qkv.N == (d.heads + 2 * d.kv_heads) * d.head_dim, "qkv rows");
    b.o = plain_lin(arena_, m, p + "self_attn.o_proj", false, H, H, s);
    b.gateup = gateup_lin(arena_, m, p + "mlp.", false, d.inter, inter_pad_, H, s);
    b.down = plain_lin(arena_, m, p + "mlp.down_proj", false, H, d.inter, s);
  }
  final_norm_ = m.f32(arena_, "norm.weight", s);
  // Qwen2.5-VL-7B does not tie the output projection to the embedding; generate_latents never reads it, generate() does.
  if (ws.has("lm_head.weight")) lm_head_ = plain_lin(arena_, ws, "lm_head", false, d.vocab, H, s);
  N1_CUDA(cudaStreamSynchronize(s));
  loaded_ = true;
}

// ------------------------------------------------------------------------------------------------ plans
VitPlan* S2Model::make_vit_plan(const int32_t* grid, int n_img, cudaStream_t s) const {
  N1_CHECK(loaded_, "System-2 weights not loaded");
  std::unique_ptr<VitPlan> p(new VitPlan());
  vit_index(grid, n_img, dims.v_merge, dims.v_window / dims.v_merge / dims.v_patch, p->host);
  p->window_index = upload(p->host.window_index, s);
  p->reverse_index = upload(p->host.reverse_index, s);
  p->cu_window = upload(p->host.cu_window, s);
  p->cu_full = upload(p->host.cu_full, s);
  p->n_window = (int)p->host.cu_window.size() - 1;
  p->n_full = (int)p->host.cu_full.size() - 1;
  int* pos = upload(p->host.pos_hw, s);
  const int half = (dims.v_hidden / dims.v_heads) / 2;
  N1_CUDA(cudaMalloc(&p->rope, (size_t)p->host.n_patches * half * sizeof(float2)));
  vit_rope_table(pos, p->rope, p->host.n_patches, half, 10000.0f, s);
  N1_CUDA(cudaStreamSynchronize(s));
  cudaFree(pos);
  return p.release();
}

KvPool::~KvPool() { cudaFree(k), cudaFree(v), cudaFree(table); }

KvPool* S2Model::make_pool(int slots, int cap) const {
  N1_CHECK(loaded_, "System-2 weights not loaded");
  N1_CHECK(slots > 0 && cap > 0 && (long)slots * cap < (1L << 31), "kv pool: slots and capacity must be positive");
  std::unique_ptr<KvPool> p(new KvPool());
  p->slots = slots, p->cap = cap, p->layers = dims.layers, p->width = dims.kv_heads * dims.head_dim;
  p->layer_stride = (long)slots * cap * p->width;
  p->valid.assign(slots, 0);
  N1_CUDA(cudaMalloc(&p->k, (size_t)p->layer_stride * dims.layers * sizeof(bf16)));
  N1_CUDA(cudaMalloc(&p->v, (size_t)p->layer_stride * dims.layers * sizeof(bf16)));
  return p.release();
}

KvPool* S2Model::make_paged_pool(int slots, int pages, int max_tokens) const {
  N1_CHECK(loaded_, "System-2 weights not loaded");
  N1_CHECK(slots > 0 && pages > 0 && max_tokens > 0, "kv pool: slots, pages and tokens per slot must be positive");
  const int per_slot = (max_tokens + kPageRows - 1) / kPageRows;
  N1_CHECK((long)slots * per_slot * kPageRows < (1L << 31), "kv pool: slots x tokens per slot must stay below 2^31");
  std::unique_ptr<KvPool> p(new KvPool());
  p->pages.init(slots, per_slot, pages);
  p->slots = slots, p->cap = per_slot * kPageRows, p->max_tokens = max_tokens;
  p->layers = dims.layers, p->width = dims.kv_heads * dims.head_dim;
  p->layer_stride = (long)pages * kPageRows * p->width;
  p->valid.assign(slots, 0);
  N1_CUDA(cudaMalloc(&p->k, (size_t)p->layer_stride * dims.layers * sizeof(bf16)));
  N1_CUDA(cudaMalloc(&p->v, (size_t)p->layer_stride * dims.layers * sizeof(bf16)));
  N1_CUDA(cudaMalloc(&p->table, p->pages.table.size() * sizeof(int)));
  N1_CUDA(cudaMemcpy(p->table, p->pages.table.data(), p->pages.table.size() * sizeof(int), cudaMemcpyHostToDevice));
  return p.release();
}

LlmPlan* S2Model::make_llm_plan(const int32_t* ids, const int32_t* lens, int B, const int32_t* grid, int n_img,
                                cudaStream_t s, int max_new_tokens, const int32_t* ctx_in, const int32_t* slot_in,
                                KvPool* pool) const {
  N1_CHECK(loaded_, "System-2 weights not loaded");
  N1_CHECK(max_new_tokens >= 0, "llm plan: max_new_tokens must be >= 0");
  const bool cont = pool != nullptr;
  N1_CHECK(cont == (ctx_in != nullptr) && cont == (slot_in != nullptr), "continuation plan: ctx, slots and pool go together");
  N1_CHECK(!cont || max_new_tokens > 0, "continuation plan: only generation plans continue a cache");
  if (max_new_tokens == 0 && !has_latent_queries())
    throw Error(-6, "latent plan: its prompts end in TRAJ tokens, and latent_queries was not part of the loaded state_dict "
                    "(a System-2-only model)");
  std::unique_ptr<LlmPlan> p(new LlmPlan());
  PlanArgs a;
  a.merge = dims.v_merge, a.vocab = dims.vocab, a.n_query = dims.n_query, a.max_new = max_new_tokens;
  a.ctx = ctx_in, a.slots = slot_in;
  if (cont) a.pool_slots = pool->slots, a.pool_cap = pool->cap, a.pool_limit = pool->max_tokens;
  PlanRows r;
  plan_rows(ids, lens, B, grid, n_img, a, r);
  p->B = B, p->n_query = dims.n_query, p->pool = pool;
  p->h_cu = std::move(r.cu), p->h_pos3 = std::move(r.pos3), p->h_delta = std::move(r.delta);
  p->tokens = p->h_cu.back();
  p->n_image_tokens = r.n_image_tokens;
  p->n_out = (int)r.out_rows.size();
  p->max_len = r.max_len;
  if (max_new_tokens > 0) p->max_new = max_new_tokens, p->slot = r.slot;
  if (cont) p->h_ctx = r.ctx, p->h_slot = r.slot_of, p->h_len = r.len, p->any_ctx = r.any_ctx;
  const int half = dims.head_dim / 2;
  // one pooled block: [ints: cu | kind | src | out_rows | pos3 | dest | len | delta | ctx | row0] [rope table]; one H2D
  // copy from the block's pinned twin, one kernel, no allocation / free / synchronisation once the pool holds a block of
  // this size
  constexpr int kParts = 10;
  const std::vector<int>* parts[kParts] = {&p->h_cu, &r.kind, &r.src, &r.out_rows, &p->h_pos3, &r.dest, &r.len, &p->h_delta,
                                           &r.ctx, &r.row0};
  size_t off_i[kParts + 1] = {0};
  for (int i = 0; i < kParts; ++i) off_i[i + 1] = off_i[i] + ((parts[i]->size() + 3) & ~size_t(3));  // 16-byte aligned
  const size_t int_bytes = (off_i[kParts] * sizeof(int) + 255) & ~size_t(255);
  const size_t need = int_bytes + (size_t)p->tokens * half * sizeof(float2);
  PlanBlock blk = pool_take(need);
  p->block = blk.dev, p->block_bytes = blk.bytes, p->last_use = blk.last_use;
  {
    std::lock_guard<std::mutex> lk(g_twin.mu);
    g_twin.map.emplace_back(blk.dev, blk.host);
  }
  N1_CUDA(cudaStreamWaitEvent(s, blk.last_use, 0));  // the previous owner's consumers (any stream) are done before we overwrite
  N1_CUDA(cudaEventSynchronize(blk.last_use));       // ... and before the pinned twin is rewritten (no-op unless just recycled)
  int* hp = static_cast<int*>(blk.host);
  for (int i = 0; i < kParts; ++i)
    if (!parts[i]->empty()) memcpy(hp + off_i[i], parts[i]->data(), parts[i]->size() * sizeof(int));
  N1_CUDA(cudaMemcpyAsync(blk.dev, blk.host, off_i[kParts] * sizeof(int), cudaMemcpyHostToDevice, s));
  int* dp = static_cast<int*>(blk.dev);
  p->cu = dp + off_i[0], p->kind = dp + off_i[1], p->src = dp + off_i[2], p->out_rows = dp + off_i[3];
  int* pos = dp + off_i[4];
  if (max_new_tokens > 0) p->dest_rows = dp + off_i[5], p->d_len = dp + off_i[6], p->d_delta = dp + off_i[7];
  if (cont) p->ctx = dp + off_i[8], p->row0 = dp + off_i[9];
  p->rope = reinterpret_cast<float2*>(static_cast<uint8_t*>(blk.dev) + int_bytes);
  mrope_table(pos, p->rope, p->tokens, half, dims.mrope[0], dims.mrope[1], dims.rope_theta, s);
  N1_CUDA(cudaEventCreateWithFlags(&p->ready, cudaEventDisableTiming));
  N1_CUDA(cudaEventRecord(p->ready, s));
  N1_CUDA(cudaEventRecord(p->last_use, s));  // a plan that is never consumed still leaves its block in a defined state
  return p.release();
}

// ------------------------------------------------------------------------------------------------ transformer block
void S2Model::block_in(const Block& b, const bf16* x, bf16* ln, bf16* qkv, const float2* rope, int rows, int H,
                       int rot_heads, int hd, float eps, cudaStream_t s) {
  layernorm(x, H, ln, H, b.n1, nullptr, rows, H, eps, 1, s);
  linear(b.qkv, ln, H, qkv, b.qkv.N, rows, GemmEpilogue(), s);
  apply_rope(qkv, b.qkv.N, rope, rows, rot_heads, hd, s);  // q and k are adjacent column blocks
}

void S2Model::block_out(const Block& b, const bf16* att, bf16* x, bf16* ln, bf16* hid, int rows, int H, int inter_pad,
                        float eps, cudaStream_t s, bf16* save_mid) {
  GemmEpilogue res;
  res.residual = x, res.ldr = H;
  linear(b.o, att, H, x, H, rows, res, s);
  if (save_mid) N1_CUDA(cudaMemcpyAsync(save_mid, x, (size_t)rows * H * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
  layernorm(x, H, ln, H, b.n2, nullptr, rows, H, eps, 1, s);
  GemmEpilogue sw;
  sw.act = ACT_SWIGLU;
  linear(b.gateup, ln, H, hid, inter_pad, rows, sw, s);
  linear(b.down, hid, inter_pad, x, H, rows, res, s);
}

// ------------------------------------------------------------------------------------------------ vision tower
size_t S2Model::vit_impl(Carver c, const VitPlan& p, const bf16* pixels, bf16* out, cudaStream_t s,
                         const int32_t* dst_rows_host) const {
  const int Hv = dims.v_hidden, unit = dims.v_merge * dims.v_merge;
  const long N = p.host.n_patches, Nm = N / unit;
  bf16* xin = c.take<bf16>(N * patch_k_);
  bf16* x = c.take<bf16>(N * Hv);
  bf16* ln = c.take<bf16>(N * Hv);
  bf16* qkv = c.take<bf16>(N * 3 * Hv);
  bf16* att = c.take<bf16>(N * Hv);
  bf16* hid = c.take<bf16>(N * (long)std::max(v_inter_pad_, Hv));
  bf16* m2 = c.take<bf16>(Nm * dims.v_out);
  int* dst_rows = c.take<int>(Nm);  // last, so the buffers above sit where they sit without a row map
  if (c.dry()) return c.used();
  if (dst_rows_host)
    N1_CUDA(cudaMemcpyAsync(dst_rows, dst_rows_host, Nm * sizeof(int), cudaMemcpyHostToDevice, s));

  gather_rows(pixels, p.window_index, xin, N, unit, patch_k_, s);  // hidden_states[window_index] on merge groups
  linear(v_patch_, xin, patch_k_, x, Hv, (int)N, GemmEpilogue(), s);
  for (int l = 0; l < dims.v_depth; ++l) {
    block_in(vblk_[l], x, ln, qkv, p.rope, (int)N, Hv, 2 * dims.v_heads, 80, 1e-6f, s);
    bool full = false;
    for (int i = 0; i < dims.n_fullatt; ++i) full |= dims.fullatt[i] == l;
    AttnParams a = {};
    a.q = qkv, a.k = qkv + Hv, a.v = qkv + 2 * Hv, a.o = att;
    a.ldq = a.ldk = a.ldv = 3 * Hv, a.ldo = Hv;
    a.heads_q = a.heads_kv = dims.v_heads, a.hd = 80;
    a.batch = full ? p.n_full : p.n_window;
    a.cu_q = a.cu_k = full ? p.cu_full : p.cu_window;
    a.max_seq_q = full ? p.host.max_full : p.host.max_window;
    a.kv_div = 1, a.scale = 1.0f / sqrtf(80.f);
    attention(a, s);
    block_out(vblk_[l], att, x, ln, hid, (int)N, Hv, v_inter_pad_, 1e-6f, s);
  }
  // merger: RMSNorm over Hv, then groups of merge^2 patches concatenated (a pure view), MLP with exact GELU
  layernorm(x, Hv, ln, Hv, merger_ln_, nullptr, (int)N, Hv, 1e-6f, 1, s);
  GemmEpilogue ge;
  ge.act = ACT_GELU;
  linear(merger0_, ln, Hv * unit, hid, Hv * unit, (int)Nm, ge, s);
  linear(merger2_, hid, Hv * unit, m2, dims.v_out, (int)Nm, GemmEpilogue(), s);
  // merged[argsort(window_index)], row r to out[dst_rows[r]] with a row map
  gather_rows(m2, p.reverse_index, out, Nm, 1, dims.v_out, s, dst_rows_host ? dst_rows : nullptr);
  return c.used();
}

size_t S2Model::ws_vit(const VitPlan& p) const { return vit_impl(Carver(nullptr, 0), p, nullptr, nullptr, nullptr); }
void S2Model::vit_forward(const VitPlan& p, void* ws, size_t ws_bytes, const bf16* pixels, bf16* out, cudaStream_t s,
                          const int32_t* dst_rows_host) const {
  N1_CHECK(loaded_ && ws, "vit_forward: not loaded / null workspace");
  if (ws_bytes < ws_vit(p)) throw Error(-7, "vit_forward: workspace too small");
  vit_impl(Carver(ws, ws_bytes), p, pixels, out, s, dst_rows_host);
}

// ------------------------------------------------------------------------------------------------ decoder prefill
size_t S2Model::llm_impl(Carver c, const LlmPlan& p, const bf16* image_feats, bf16* out, cudaStream_t s,
                         const KvCache* kv, const int32_t* image_rows_host) const {
  const int H = dims.hidden, hd = dims.head_dim;
  const long T = p.tokens;
  const int qkv_n = (dims.heads + 2 * dims.kv_heads) * hd;
  bf16* x = c.take<bf16>(T * H);
  const long sel_rows = 3L * p.n_out;  // the last layer reuses `ln` for three [n_out, H] buffers
  bf16* ln = c.take<bf16>((T > sel_rows ? T : sel_rows) * H);
  bf16* qkv = c.take<bf16>(T * qkv_n);
  bf16* att = c.take<bf16>(T * H);
  bf16* hid = c.take<bf16>(T * (long)inter_pad_);
  int* image_rows = c.take<int>(p.n_image_tokens);  // last, so the buffers above sit where they sit without a row table
  const KvPool* paged = kv && p.pool && p.pool->paged() ? p.pool : nullptr;
  int* dest_paged = paged ? c.take<int>(T) : nullptr;  // the plan's K/V rows mapped through the page table
  if (c.dry()) return c.used();

  if (image_rows_host && p.n_image_tokens > 0)
    N1_CUDA(cudaMemcpyAsync(image_rows, image_rows_host, p.n_image_tokens * sizeof(int), cudaMemcpyHostToDevice, s));
  build_embeds(p.kind, p.src, embed_, image_feats, latentq_, x, T, H, s, image_rows_host ? image_rows : nullptr);
  const int* dest = p.dest_rows;
  if (paged) page_rows(p.dest_rows, paged->table, dest_paged, T, s), dest = dest_paged;
  for (int l = 0; l < dims.layers; ++l) {
    const Block& b = lblk_[l];
    block_in(b, x, ln, qkv, p.rope, (int)T, H, dims.heads + dims.kv_heads, hd, dims.rms_eps, s);
    if (kv)  // keep the rotated keys and the values of every prompt token for the decode passes
      kv_append(qkv, qkv_n, dims.heads * hd, (dims.heads + dims.kv_heads) * hd, dims.kv_heads * hd, dest, T,
                kv->k + l * kv->layer_stride, kv->v + l * kv->layer_stride, s);
    if (p.any_ctx) {  // continued sequences: the chunk attends to its slot's cached rows (which now include its own)
      CacheAttnParams a = {};
      a.q = qkv, a.ldq = qkv_n, a.q_rows = T;
      a.k = kv->k + l * kv->layer_stride, a.v = kv->v + l * kv->layer_stride, a.ldkv = dims.kv_heads * hd;
      a.kv_rows = p.pool->rows();
      a.pages = paged ? paged->table : nullptr;
      a.o = att, a.ldo = H;
      a.cu_q = p.cu, a.ctx = p.ctx, a.row0 = p.row0;
      a.batch = p.B, a.max_chunk = p.max_len, a.heads_q = dims.heads, a.heads_kv = dims.kv_heads;
      a.scale = 1.0f / sqrtf((float)hd);
      attention_cache(a, s);
    } else {
      AttnParams a = {};
      a.q = qkv, a.k = qkv + (long)dims.heads * hd, a.v = qkv + (long)(dims.heads + dims.kv_heads) * hd, a.o = att;
      a.ldq = a.ldk = a.ldv = qkv_n, a.ldo = H;
      a.heads_q = dims.heads, a.heads_kv = dims.kv_heads, a.hd = hd;
      a.batch = p.B, a.cu_q = a.cu_k = p.cu, a.max_seq_q = p.max_len, a.total_rows = T;
      a.kv_div = 1, a.causal = 1, a.scale = 1.0f / sqrtf((float)hd);
      attention(a, s);
    }
    if (l == dims.layers - 1) {
      // Only the n_query TRAJ rows of each sequence are read after the last layer (internvla_n1.py L345): every token
      // still contributes K/V to the attention above, but o_proj and the MLP run on those B * n_query rows alone.
      // (Generation plans read the last prompt row of each sequence instead.)
      const int R = p.n_out;
      bf16* att_sel = ln;                      // [R, H] scratch (ln is free here)
      bf16* x_sel = ln + (long)R * H;          // [R, H]
      bf16* ln_sel = ln + 2L * R * H;          // [R, H]
      gather_rows(att, p.out_rows, att_sel, R, 1, H, s);
      gather_rows(x, p.out_rows, x_sel, R, 1, H, s);
      block_out(b, att_sel, x_sel, ln_sel, hid, R, H, inter_pad_, dims.rms_eps, s);
      // outputs.hidden_states[-1][:, -N_QUERY:, :] -- the last entry is post final-norm
      layernorm(x_sel, H, out, H, final_norm_, nullptr, R, H, dims.rms_eps, 1, s);
      break;
    }
    block_out(b, att, x, ln, hid, (int)T, H, inter_pad_, dims.rms_eps, s);
  }
  return c.used();
}

size_t S2Model::ws_llm(const LlmPlan& p) const { return llm_impl(Carver(nullptr, 0), p, nullptr, nullptr, nullptr); }
void S2Model::llm_prefill(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* image_feats, bf16* out,
                          cudaStream_t s) const {
  N1_CHECK(loaded_ && ws, "llm_prefill: not loaded / null workspace");
  N1_CHECK(p.max_new == 0, "llm_prefill: this is a generation plan (use llm_generate)");
  if (!has_latent_queries()) throw Error(-6, "llm_prefill: latent_queries was not part of the loaded state_dict");
  if (ws_bytes < ws_llm(p)) throw Error(-7, "llm_prefill: workspace too small");
  p.wait_ready(s);
  llm_impl(Carver(ws, ws_bytes), p, image_feats, out, s);
  p.mark_used(s);
}

// ------------------------------------------------------------------------------------------------ greedy decode
AttnParams S2Model::cache_attn(const LlmPlan& p, int per_seq, const int* k_len, const bf16* qkv, const bf16* k,
                               const bf16* v, bf16* o) const {
  const int hd = dims.head_dim;
  AttnParams a = {};
  a.q = qkv, a.k = k, a.v = v, a.o = o;
  a.ldq = (dims.heads + 2 * dims.kv_heads) * hd, a.ldk = a.ldv = dims.kv_heads * hd, a.ldo = dims.hidden;
  a.heads_q = dims.heads, a.heads_kv = dims.kv_heads, a.hd = hd;
  a.batch = p.B, a.seq_q = per_seq, a.k_len = k_len, a.k_slot = p.slot, a.k_row0 = p.row0;
  a.k_pages = p.pool && p.pool->paged() ? p.pool->table : nullptr;
  a.kv_div = 1, a.causal = 1, a.scale = 1.0f / sqrtf((float)hd);
  return a;
}

// One pass of B * per_seq new tokens (rows of g.x) through all layers against the cache: per_seq = 1 is a decode step,
// per_seq = 1 + n_query the latent pass, per_seq = n_query the training forward.  g.dest / g.rope / g.k_len describe the
// chunk (gen_rows).  Result: final-norm states of every row in g.normed, the last residual stream in g.x.  With `save`
// each layer's input, q|k|v, attention output and post-attention residual go to its per-layer arrays, and g.qkv / g.att
// are not used.
void S2Model::chunk_pass(const GenBufs& g, const LlmPlan& p, const KvCache& kv, int per_seq, cudaStream_t s,
                         const ChunkSaves* save) const {
  const int H = dims.hidden, hd = dims.head_dim, R = p.B * per_seq;
  const int qkv_n = (dims.heads + 2 * dims.kv_heads) * hd, kvd = dims.kv_heads * hd;
  for (int l = 0; l < dims.layers; ++l) {
    const Block& b = lblk_[l];
    bf16* qkv = save ? save->qkv + (size_t)l * R * qkv_n : g.qkv;
    bf16* att = save ? save->att + (size_t)l * R * H : g.att;
    if (save)
      N1_CUDA(cudaMemcpyAsync(save->x_in + (size_t)l * R * H, g.x, (size_t)R * H * sizeof(bf16), cudaMemcpyDeviceToDevice,
                              s));
    block_in(b, g.x, g.ln, qkv, g.rope, R, H, dims.heads + dims.kv_heads, hd, dims.rms_eps, s);
    bf16* ck = kv.k + l * kv.layer_stride;
    bf16* cv = kv.v + l * kv.layer_stride;
    kv_append(qkv, qkv_n, dims.heads * hd, (dims.heads + dims.kv_heads) * hd, kvd, g.dest, R, ck, cv, s);
    attention(cache_attn(p, per_seq, g.k_len, qkv, ck, cv, att), s);
    block_out(b, att, g.x, g.ln, g.hid, R, H, inter_pad_, dims.rms_eps, s,
              save ? save->x_mid + (size_t)l * R * H : nullptr);
  }
  layernorm(g.x, H, g.normed, H, final_norm_, nullptr, R, H, dims.rms_eps, 1, s);
}

size_t S2Model::gen_impl(Carver c, const LlmPlan& p, const bf16* image_feats, const int32_t* eos, int n_eos,
                         int32_t pad, GenResult* out, bf16* latents, cudaStream_t s,
                         const int32_t* image_rows_host) const {
  const int H = dims.hidden, hd = dims.head_dim, B = p.B, nq = dims.n_query;
  const int qkv_n = (dims.heads + 2 * dims.kv_heads) * hd, kvd = dims.kv_heads * hd, half = hd / 2;
  const int R5 = B * (nq + 1);
  const int* pages = p.pool && p.pool->paged() ? p.pool->table : nullptr;
  KvCache kv;
  if (p.pool) {  // continuation plan: the caller's pool is the cache
    kv.k = p.pool->k, kv.v = p.pool->v, kv.layer_stride = p.pool->layer_stride;
  } else {
    kv.layer_stride = (long)B * p.slot * kvd;
    kv.k = c.take<bf16>((size_t)dims.layers * kv.layer_stride);
    kv.v = c.take<bf16>((size_t)dims.layers * kv.layer_stride);
  }
  GenBufs g;
  g.cur_tok = c.take<int>(B), g.gen = c.take<int>(B), g.finished = c.take<int>(B), g.next = c.take<int>(B);
  g.k_len = c.take<int>(B), g.n_active = c.take<int>(1), g.out_tokens = c.take<int>((size_t)B * p.max_new);
  g.dest = c.take<int>(R5), g.pos3 = c.take<int>(3 * R5), g.kind = c.take<int>(R5), g.src = c.take<int>(R5);
  g.rope = c.take<float2>((size_t)R5 * half);
  g.x = c.take<bf16>((size_t)R5 * H), g.ln = c.take<bf16>((size_t)R5 * H), g.qkv = c.take<bf16>((size_t)R5 * qkv_n);
  g.att = c.take<bf16>((size_t)R5 * H), g.hid = c.take<bf16>((size_t)R5 * inter_pad_);
  g.normed = c.take<bf16>((size_t)R5 * H), g.logits = c.take<bf16>((size_t)B * dims.vocab);
  if (c.dry()) return llm_impl(c, p, nullptr, nullptr, nullptr, &kv);  // prefill scratch follows the decode state

  // 1. prompt prefill, K/V kept; final-norm state of the last prompt token of each sequence -> g.normed [B, H]
  llm_impl(c, p, image_feats, g.normed, s, &kv, image_rows_host);
  std::vector<int32_t> fill((size_t)B * p.max_new, pad);
  N1_CUDA(cudaMemcpyAsync(g.out_tokens, fill.data(), fill.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  N1_CUDA(cudaMemsetAsync(g.gen, 0, B * sizeof(int), s));
  N1_CUDA(cudaMemsetAsync(g.finished, 0, B * sizeof(int), s));
  int steps = 0;
  for (int it = 0; it < p.max_new; ++it) {
    // logits = lm_head(hidden[:, -1]) in bf16, next = argmax (GenerationMixin greedy search)
    linear(lm_head_, g.normed, H, g.logits, dims.vocab, B, GemmEpilogue(), s);
    argmax_rows(g.logits, dims.vocab, dims.vocab, B, g.next, s);
    gen_update(g.next, g.cur_tok, g.gen, g.finished, g.out_tokens, p.max_new, eos, n_eos, B, g.n_active, s);
    int active = 0;
    N1_CUDA(cudaMemcpyAsync(&active, g.n_active, sizeof(int), cudaMemcpyDeviceToHost, s));
    N1_CUDA(cudaStreamSynchronize(s));
    if (active == 0) break;
    // 2. one decode pass: the token just sampled is row (len + gen - 1) of its sequence
    gen_rows(p.d_len, p.d_delta, g.gen, 1, 1, B, p.slot, p.row0, pages, g.dest, g.pos3, g.k_len, s);
    mrope_table(g.pos3, g.rope, B, half, dims.mrope[0], dims.mrope[1], dims.rope_theta, s);
    gather_rows(embed_, g.cur_tok, g.x, B, 1, H, s);
    chunk_pass(g, p, kv, 1, s);
    ++steps;
  }
  if (latents) {
    // 3. generate_latents(output_ids, ...) on the cache: the last sampled token has no K/V yet, so the pass covers
    //    [last token, TRAJ x nq]; rows 1..nq of each sequence are the latent plan (internvla_n1.py L327, L345).
    gen_rows(p.d_len, p.d_delta, g.gen, 1, nq + 1, B, p.slot, p.row0, pages, g.dest, g.pos3, g.k_len, s);
    mrope_table(g.pos3, g.rope, R5, half, dims.mrope[0], dims.mrope[1], dims.rope_theta, s);
    latent_src(g.cur_tok, B, nq, g.kind, g.src, s);
    build_embeds(g.kind, g.src, embed_, nullptr, latentq_, g.x, R5, H, s);
    chunk_pass(g, p, kv, nq + 1, s);
    N1_CUDA(cudaMemcpy2DAsync(latents, (size_t)nq * H * sizeof(bf16), g.normed + H, (size_t)(nq + 1) * H * sizeof(bf16),
                              (size_t)nq * H * sizeof(bf16), B, cudaMemcpyDeviceToDevice, s));
  }
  N1_CUDA(cudaMemcpyAsync(out->tokens, g.out_tokens, (size_t)B * p.max_new * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  N1_CUDA(cudaMemcpyAsync(out->lens, g.gen, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  N1_CUDA(cudaStreamSynchronize(s));
  out->steps = steps;
  return c.used();
}

size_t S2Model::ws_generate(const LlmPlan& p) const {
  N1_CHECK(p.max_new > 0, "ws_generate: not a generation plan");
  return gen_impl(Carver(nullptr, 0), p, nullptr, nullptr, 0, 0, nullptr, nullptr, nullptr);
}
void S2Model::llm_generate(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* image_feats, const int32_t* eos,
                           int n_eos, int32_t pad, GenResult& out, bf16* latents, cudaStream_t s,
                           const int32_t* image_rows_host) const {
  N1_CHECK(loaded_ && ws, "llm_generate: not loaded / null workspace");
  N1_CHECK(p.max_new > 0, "llm_generate: the plan was not created for generation");
  if (!has_lm_head()) throw Error(-6, "llm_generate: lm_head.weight was not part of the loaded state_dict");
  if (latents && !has_latent_queries())
    throw Error(-6, "llm_generate: latents requested, but latent_queries was not part of the loaded state_dict");
  N1_CHECK(out.tokens && out.lens, "llm_generate: null output buffers");
  KvPool* pool = p.pool;
  if (pool)
    for (int b = 0; b < p.B; ++b)
      N1_CHECK(p.h_ctx[b] <= pool->valid[p.h_slot[b]],
               "llm_generate: sequence " + std::to_string(b) + " reuses " + std::to_string(p.h_ctx[b]) +
                   " rows but slot " + std::to_string(p.h_slot[b]) + " holds " + std::to_string(pool->valid[p.h_slot[b]]));
  if (ws_bytes < ws_generate(p)) throw Error(-7, "llm_generate: workspace too small");
  if (pool && pool->paged()) {
    // each sequence keeps the pages of its reused prefix and holds pages for every row the call may write; refused
    // (N1_ERR_KV_PAGES, nothing launched, the pool unchanged) when the free pages do not cover that
    std::vector<int32_t> need(p.B);
    for (int b = 0; b < p.B; ++b) need[b] = p.h_len[b] + p.max_new + p.n_query;
    const std::pair<int, int> ch = pool->pages.prepare(p.B, p.h_slot.data(), p.h_ctx.data(), need.data());
    const size_t row = pool->pages.per_slot;
    if (ch.first < ch.second)
      N1_CUDA(cudaMemcpyAsync(pool->table + ch.first * row, pool->pages.table.data() + ch.first * row,
                              (ch.second - ch.first) * row * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  if (pool)  // rows past ctx are rewritten from here on
    for (int b = 0; b < p.B; ++b) pool->valid[p.h_slot[b]] = p.h_ctx[b];
  p.wait_ready(s);
  gen_impl(Carver(ws, ws_bytes), p, image_feats, eos, n_eos, pad, &out, latents, s, image_rows_host);
  p.mark_used(s);
  // K/V exist for the prompt and every generated token but the last; the latent pass writes the last one too (and the
  // TRAJ rows after it, which are not part of the conversation)
  if (pool)
    for (int b = 0; b < p.B; ++b) {
      const int slot = p.h_slot[b];
      pool->valid[slot] = p.h_len[b] + out.lens[b] - (latents ? 0 : 1);
      if (pool->paged()) pool->pages.trim(slot, pool->valid[slot]);  // the TRAJ rows and the unused budget
    }
}

}  // namespace n1
