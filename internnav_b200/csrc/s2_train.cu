// Training branch, System-2 half: TRAJ-row forward on the prompt's K/V cache and its backward to latent_queries.
// Algorithm and parity target: oracle/qwen_backward.py (equal to autograd through the padded-batch forward).
#include <algorithm>

#include "bwd_kernels.h"
#include "s2_kernels.h"
#include "s2_model.h"

namespace n1 {

namespace {

inline int nblk(long n) { return (int)((n + 255) / 256); }

__global__ void fill_latent_rows_kernel(int* kind, int* src, int rows, int nq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  kind[i] = 2, src[i] = i % nq;
}

// the TRAJ columns of dK / dV (fp32, cache-row indexed) -> the K / V column blocks of the packed dqkv rows (bf16)
__global__ void gather_kv_grad_kernel(const float* __restrict__ dk, const float* __restrict__ dv,
                                      const int* __restrict__ dest, int rows, int kvd, bf16* __restrict__ dqkv, int ld,
                                      int k_off, int v_off) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)rows * kvd) return;
  const int r = i / kvd, c = i % kvd;
  const long srow = (long)dest[r] * kvd + c;
  dqkv[(long)r * ld + k_off + c] = __float2bfloat16(dk[srow]);
  dqkv[(long)r * ld + v_off + c] = __float2bfloat16(dv[srow]);
}

// out[j, c] = sum_b d[b * nq + j, c]
__global__ void sum_over_batch_kernel(const bf16* __restrict__ d, int B, int nq, int H, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)nq * H) return;
  const int j = i / H, c = i % H;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += __bfloat162float(d[((long)b * nq + j) * H + c]);
  out[i] = acc;
}

Lin transposed(Arena& a, const Lin& L, cudaStream_t s) {
  Lin T;
  T.N = L.K, T.K = (L.N + 7) & ~7, T.ldw = T.K;  // out = A @ T.w^T with T.w [K_orig, N_orig]: dX = dY @ W
  T.w = a.alloc_n<bf16>((size_t)T.N * T.ldw);
  transpose_bf16(L.w, L.N, L.K, L.ldw, T.w, T.ldw, T.K, s);
  return T;
}

}  // namespace

struct S2Model::TrainBufs {
  KvCache kv;
  GenBufs g;        // the TRAJ chunk: its row description and forward scratch; g.x ends as the last residual stream
  ChunkSaves save;  // per-layer saves: [layers][R, .]
  bf16 *d, *pre, *dpre, *dact, *da, *dqkv, *dh;     // backward scratch
  float *dk, *dv;                                    // [B * slot, kvd] fp32
  int R;
};

void S2Model::ensure_transposed(cudaStream_t s) {
  if (!lblk_t_.empty()) return;
  lblk_t_.resize(dims.layers);
  for (int l = 0; l < dims.layers; ++l) {
    lblk_t_[l].qkv = transposed(arena_, lblk_[l].qkv, s);
    lblk_t_[l].o = transposed(arena_, lblk_[l].o, s);
    lblk_t_[l].gateup = transposed(arena_, lblk_[l].gateup, s);
    lblk_t_[l].down = transposed(arena_, lblk_[l].down, s);
  }
  N1_CUDA(cudaStreamSynchronize(s));
}

size_t S2Model::train_carve(Carver& c, const LlmPlan& p, TrainBufs& t) const {
  const int H = dims.hidden, hd = dims.head_dim, B = p.B, nq = dims.n_query, L = dims.layers;
  const int qkv_n = (dims.heads + 2 * dims.kv_heads) * hd, kvd = dims.kv_heads * hd;
  const int R = B * nq;
  t.R = R;
  t.kv.layer_stride = (long)B * p.slot * kvd;
  t.kv.k = c.take<bf16>((size_t)L * t.kv.layer_stride);
  t.kv.v = c.take<bf16>((size_t)L * t.kv.layer_stride);
  GenBufs& g = t.g;
  g.gen = c.take<int>(B), g.k_len = c.take<int>(B), g.dest = c.take<int>(R), g.pos3 = c.take<int>(3 * R);
  g.kind = c.take<int>(R), g.src = c.take<int>(R);
  g.rope = c.take<float2>((size_t)R * (hd / 2));
  t.save.x_in = c.take<bf16>((size_t)L * R * H), t.save.qkv = c.take<bf16>((size_t)L * R * qkv_n);
  t.save.att = c.take<bf16>((size_t)L * R * H), t.save.x_mid = c.take<bf16>((size_t)L * R * H);
  g.x = c.take<bf16>((size_t)R * H), g.ln = c.take<bf16>((size_t)R * H), g.hid = c.take<bf16>((size_t)R * inter_pad_);
  t.d = c.take<bf16>((size_t)R * H), t.pre = c.take<bf16>((size_t)R * 2 * inter_pad_);
  t.dpre = c.take<bf16>((size_t)R * 2 * inter_pad_), t.dact = c.take<bf16>((size_t)R * inter_pad_);
  t.da = c.take<bf16>((size_t)R * H), t.dqkv = c.take<bf16>((size_t)R * qkv_n), t.dh = c.take<bf16>((size_t)R * H);
  t.dk = c.take<float>((size_t)B * p.slot * kvd), t.dv = c.take<float>((size_t)B * p.slot * kvd);
  return c.used();
}

void S2Model::set_latent_queries(const bf16* src, cudaStream_t s) {
  N1_CHECK(loaded_ && src, "set_latent_queries: not loaded / null source");
  if (!has_latent_queries()) throw Error(-6, "set_latent_queries: latent_queries was not part of the loaded state_dict");
  N1_CUDA(cudaMemcpyAsync(latentq_, src, (size_t)dims.n_query * dims.hidden * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
}

size_t S2Model::ws_train(const LlmPlan& p) const {
  // a continuation plan's dest_rows index pool rows (slot * pool_cap + ...), which lie outside the B * slot rows per
  // layer of the workspace's cache
  N1_CHECK(!p.pool, "training: the plan continues a K/V pool; training needs a generation plan created without a pool");
  N1_CHECK(p.max_new > 0, "ws_train: needs a generation plan (prompts without TRAJ tokens)");
  Carver c(nullptr, 0);
  TrainBufs t;
  train_carve(c, p, t);
  return llm_impl(c, p, nullptr, nullptr, nullptr, &t.kv);  // the prefill scratch follows
}

void S2Model::train_forward(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* image_feats, bf16* states,
                            cudaStream_t s) {
  N1_CHECK(loaded_ && ws && states, "train_forward: not loaded / null buffers");
  if (!has_latent_queries()) throw Error(-6, "train_forward: latent_queries was not part of the loaded state_dict");
  N1_CHECK(p.max_new > 0 && p.slot >= p.max_len + dims.n_query, "train_forward: needs a generation plan");
  if (ws_bytes < ws_train(p)) throw Error(-7, "train_forward: workspace too small");
  p.wait_ready(s);
  const int H = dims.hidden, hd = dims.head_dim, nq = dims.n_query;
  Carver c(ws, ws_bytes);
  TrainBufs t;
  train_carve(c, p, t);
  GenBufs& g = t.g;
  const int R = t.R;
  // 1. prompt prefill with the K/V of every layer kept (the value it returns -- last prompt row -- is not needed)
  llm_impl(c, p, image_feats, g.ln, s, &t.kv);
  // 2. the n_query TRAJ rows of every sample as one chunk on that cache: rows len .. len + n_query - 1
  N1_CUDA(cudaMemsetAsync(g.gen, 0, p.B * sizeof(int), s));
  gen_rows(p.d_len, p.d_delta, g.gen, 0, nq, p.B, p.slot, nullptr, nullptr, g.dest, g.pos3, g.k_len, s);
  mrope_table(g.pos3, g.rope, R, hd / 2, dims.mrope[0], dims.mrope[1], dims.rope_theta, s);
  fill_latent_rows_kernel<<<nblk(R), 256, 0, s>>>(g.kind, g.src, R, nq);
  N1_CUDA(cudaGetLastError());
  build_embeds(g.kind, g.src, embed_, nullptr, latentq_, g.x, R, H, s);
  g.normed = states;
  chunk_pass(g, p, t.kv, nq, s, &t.save);
  p.mark_used(s);
}

void S2Model::train_backward(const LlmPlan& p, void* ws, size_t ws_bytes, const bf16* grad_states, float* grad_latent,
                             cudaStream_t s) {
  N1_CHECK(loaded_ && ws && grad_states && grad_latent, "train_backward: not loaded / null buffers");
  if (!has_latent_queries()) throw Error(-6, "train_backward: latent_queries was not part of the loaded state_dict");
  if (ws_bytes < ws_train(p)) throw Error(-7, "train_backward: workspace too small");
  p.wait_ready(s);
  ensure_transposed(s);
  const int H = dims.hidden, hd = dims.head_dim, nq = dims.n_query;
  const int qkv_n = (dims.heads + 2 * dims.kv_heads) * hd, kvd = dims.kv_heads * hd;
  Carver c(ws, ws_bytes);
  TrainBufs t;
  train_carve(c, p, t);
  const int R = t.R;
  const float eps = dims.rms_eps;
  const GenBufs& g = t.g;
  norm_bwd(grad_states, H, g.x, H, final_norm_, nullptr, 0, t.d, H, nullptr, nullptr, R, H, eps, 1, 0, s);
  for (int l = dims.layers - 1; l >= 0; --l) {
    const Block& b = lblk_[l];
    const Block& bt = lblk_t_[l];
    const bf16* x_in = t.save.x_in + (size_t)l * R * H;
    const bf16* x_mid = t.save.x_mid + (size_t)l * R * H;
    // MLP: recompute the gate / up pre-activations of these rows, then dgrad through down, SwiGLU, gate/up
    layernorm(x_mid, H, g.ln, H, b.n2, nullptr, R, H, eps, 1, s);
    linear(b.gateup, g.ln, H, t.pre, 2 * inter_pad_, R, GemmEpilogue(), s);
    linear(bt.down, t.d, H, t.dact, inter_pad_, R, GemmEpilogue(), s);
    swiglu_bwd(t.pre, t.dact, t.dpre, R, inter_pad_, s);
    linear(bt.gateup, t.dpre, 2 * inter_pad_, t.dh, H, R, GemmEpilogue(), s);
    norm_bwd(t.dh, H, x_mid, H, b.n2, t.d, H, t.d, H, nullptr, nullptr, R, H, eps, 1, 0, s);
    // attention: dO = d W_o ; backward of n_query queries per sample over the visible keys of the cache
    linear(bt.o, t.d, H, t.da, H, R, GemmEpilogue(), s);
    N1_CUDA(cudaMemsetAsync(t.dk, 0, (size_t)p.B * p.slot * kvd * sizeof(float), s));
    N1_CUDA(cudaMemsetAsync(t.dv, 0, (size_t)p.B * p.slot * kvd * sizeof(float), s));
    AttnBwdParams ab = {};
    ab.f = cache_attn(p, nq, g.k_len, t.save.qkv + (size_t)l * R * qkv_n, t.kv.k + l * t.kv.layer_stride,
                      t.kv.v + l * t.kv.layer_stride, t.save.att + (size_t)l * R * H);
    ab.dout = t.da, ab.lddo = H, ab.dq = t.dqkv, ab.lddq = qkv_n, ab.dk = t.dk, ab.dv = t.dv;
    attention_bwd(ab, s);
    gather_kv_grad_kernel<<<nblk((long)R * kvd), 256, 0, s>>>(t.dk, t.dv, g.dest, R, kvd, t.dqkv, qkv_n, dims.heads * hd,
                                                            (dims.heads + dims.kv_heads) * hd);
    N1_CUDA(cudaGetLastError());
    rope_transposed(t.dqkv, qkv_n, g.rope, R, dims.heads + dims.kv_heads, hd, s);
    linear(bt.qkv, t.dqkv, qkv_n, t.dh, H, R, GemmEpilogue(), s);
    norm_bwd(t.dh, H, x_in, H, b.n1, t.d, H, t.d, H, nullptr, nullptr, R, H, eps, 1, 0, s);
  }
  sum_over_batch_kernel<<<nblk((long)nq * H), 256, 0, s>>>(t.d, p.B, nq, H, grad_latent);
  N1_CUDA(cudaGetLastError());
  p.mark_used(s);
}

}  // namespace n1
